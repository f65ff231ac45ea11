"""GPU: the warp kernels on layouts whose factors follow their position-0 q row (layout.build_layout) against the
generic kernels (PYDCOP_B200_NO_FAST=1), bit for bit: hubs, several factor classes (tiles at class boundaries), sparse
graphs whose first variables are spread over q, and a sharded layout whose ghost-stub classes keep the caller's
order."""
import numpy as np
import pytest

from pydcop_b200.generators import random_factor_graph

pytestmark = pytest.mark.gpu


def _instance(n_vars, d, n_factors, seed, hubs=(), d2=None):
    rng = np.random.default_rng(seed)
    inst = random_factor_graph(n_vars, d, n_factors, 2, seed=seed)
    ev = inst["edge_var"].reshape(-1, 2).copy()
    for h in hubs:                                     # hub h is the first variable of ~3 % of the factors
        pick = rng.random(n_factors) < 0.03
        ev[pick, 0] = h
    same = ev[:, 0] == ev[:, 1]
    ev[same, 1] = (ev[same, 0] + 1) % n_vars
    inst["edge_var"] = ev.reshape(-1).astype(np.int32)
    if d2 is not None:                                 # a second domain size: a second binary factor class
        dom = inst["dom_size"].copy()
        dom[rng.random(n_vars) < 0.3] = d2
        inst["dom_size"] = dom
        sizes = dom[ev[:, 0]].astype(np.int64) * dom[ev[:, 1]]
        inst["tables"] = rng.integers(0, 9, int(sizes.sum())).astype(np.float32)
        inst.pop("table_off", None)
        if "unary" in inst:
            inst["unary"] = rng.random(int(dom.sum()))
    return inst


def _pair(monkeypatch, L, precision, cycles):
    from pydcop_b200 import MaxSumEngine
    monkeypatch.delenv("PYDCOP_B200_NO_FAST", raising=False)
    fast = MaxSumEngine(L, precision=precision).init()
    monkeypatch.setenv("PYDCOP_B200_NO_FAST", "1")
    slow = MaxSumEngine(L, precision=precision).init()
    for k in range(cycles):
        fast.step()
        slow.step()
        for a, b in zip(fast.messages(), slow.messages()):
            assert np.array_equal(a, b), k
        assert np.array_equal(fast.values()[0], slow.values()[0]), k


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("case", ["hubs", "two_classes", "sparse"])
def test_ordered_layout_warp_kernels_equal_generic_kernels(monkeypatch, case, precision):
    from pydcop_b200 import build_layout
    if case == "hubs":
        inst = _instance(4000, 10, 8000, seed=1, hubs=(3, 1700))
    elif case == "two_classes":
        inst = _instance(3000, 10, 6000, seed=2, d2=6)
    else:
        inst = _instance(6000, 10, 900, seed=3)
    L = build_layout(**inst)
    binary = [c for c in L.classes if c.arity == 2]
    assert len(binary) >= (3 if case == "two_classes" else 1), case
    for c in binary:   # ordered by the position-0 q row
        assert (np.diff(L.edge_qoff[c.first_edge:c.first_edge + 2 * c.n_factors:2]) > 0).all()
    _pair(monkeypatch, L, precision, 8)


def test_ordered_shard_layout_warp_kernels_equal_generic_kernels(monkeypatch):
    """Two shards on one device with the in-process halo of test_gpu_sharded (own classes ordered, ghost-stub classes
    in the caller's order): messages of every local edge and the owned values, warp kernels against generic ones."""
    from test_gpu_sharded import _run_sharded
    inst = _instance(5000, 10, 10000, seed=4, hubs=(11,))
    runs = []
    for no_fast in (False, True):
        if no_fast:
            monkeypatch.setenv("PYDCOP_B200_NO_FAST", "1")
        else:
            monkeypatch.delenv("PYDCOP_B200_NO_FAST", raising=False)
        shards = _run_sharded(inst, 2, 6)
        assert all(any(c.tag != 0 for c in s.plan.layout.classes) for s in shards)
        runs.append([(s.engine.messages(), s.local_values()) for s in shards])
    for (ma, va), (mb, vb) in zip(*runs):
        for a, b in zip(ma, mb):
            assert np.array_equal(a, b)
        for a, b in zip(va, vb):
            assert np.array_equal(a, b)


@pytest.mark.parametrize("precision", ["f32", "f64"])
def test_deferred_table_permutation_runs_on_the_device(precision):
    """A one-class layout in factor order uploads the caller's tables and permutes them with fg_gather_rows: the same
    array the host would have packed, and no host copy is made."""
    from pydcop_b200 import MaxSumEngine, build_layout
    inst = random_factor_graph(3000, 10, 6000, 2, seed=5)
    L = build_layout(**inst)
    assert L.table_rows is not None and L._tables is None
    eng = MaxSumEngine(L, precision=precision).init().step(3)
    assert L._tables is None
    got = eng.tables.cpu().numpy()
    want = build_layout(**inst).tables
    assert got.shape == want.shape and np.array_equal(got, want.astype(got.dtype))
