"""The MGM-2 CUDA kernel SOURCE executed on the CPU (tests/hostshim/mgm2_host.cpp runs fg_mgm2_init / fg_mgm2_step's
launch sequence from pydcop_b200/csrc/mgm2_kernels.cuh, thread after thread) with exactly the arrays Mgm2Engine
uploads, against the reference trajectories (tests/golden/mgm2_*.npz) and the oracle. This checks the kernels' logic
and the host-side array preparation without a GPU; the device run is tests/test_gpu_zz_mgm2.py's."""
import ctypes as C
import os

import numpy as np
import pytest

import _limits as LM
import oracle as orc
from _hostshim import HostRun
from _mgm2_oracle import Mgm2Oracle
from conftest import GOLDEN_DIR, golden_names
from pydcop_b200 import _cabi
from pydcop_b200.engine import mgm2_offer_offsets, mgm2_plan, mgm_host_arrays
from pydcop_b200.generators import random_factor_graph
from pydcop_b200.layout import default_var_csr, layout_from_instance
from test_mgm2_cpu import check_trajectory

P = C.c_void_p


class HostMgm2(HostRun):
    """Mgm2Engine's plan (mgm2_plan) run by tests/hostshim/mgm2_host.cpp."""

    def __init__(self, layout, precision="f64", mode="min", threshold=0.5, favor="unilateral", stop_cycle=0, seed=0,
                 var_rank=None, var_global_id=None, var_seed=None, **_):
        plan = mgm2_plan(layout, precision, mode, threshold, favor, stop_cycle, seed, var_rank,
                         var_global_id=var_global_id, var_seed=var_seed)
        super().__init__("mgm2", layout, plan, precision)
        self.nbr_ptr, self.nbr_idx = self.k["nbr_ptr"], self.k["nbr_idx"]
        self.has_nbr = np.diff(self.nbr_ptr) > 0

    def values(self):
        L, k = self.L, self.k
        cost = k["cost"][:L.n_vars].astype(np.float64)
        cost[k["has_cost"][:L.n_vars] == 0] = np.nan
        return L.vars_to_canonical(k["value"][:L.n_vars].copy()), L.vars_to_canonical(cost)

    def record(self):
        L, k, n = self.L, self.k, self.L.n_vars
        conn = self.has_nbr[:n]
        pos = np.full(n, -1, dtype=np.int32)
        for v in np.nonzero(k["partner"][:n] >= 0)[0]:
            row = self.nbr_idx[self.nbr_ptr[v]:self.nbr_ptr[v + 1]]
            pos[v] = int(np.nonzero(row == k["partner"][v])[0][0])
        out = dict(local_cost=np.where(conn, k["local_cost"][:n].astype(np.float64), np.nan),
                   gain=np.where(conn, k["gain"][:n].astype(np.float64), np.nan),
                   offerer=k["offerer"][:n].copy(), partner=pos, committed=k["committed"][:n].copy(),
                   potential_value=np.where(conn, k["potential_value"][:n], -1).astype(np.int32),
                   go=k["go"][:n].copy())
        return {key: L.vars_to_canonical(v) for key, v in out.items()}


def _assert_same(a, b, dt, k):
    for key in a:
        x, y = a[key], b[key]
        if x.dtype.kind == "f":
            assert np.array_equal(x.astype(dt), y.astype(dt), equal_nan=True), (k, key)
        else:
            assert np.array_equal(x, y), (k, key)


@pytest.mark.parametrize("name", golden_names("mgm2_"))
@pytest.mark.parametrize("precision", ["f64", "f32"])
def test_kernel_source_matches_fixture(name, precision):
    """f64 against the reference's trajectory; f32 against the f32 oracle (float fixtures round
    differently in f32) and, for integer costs, against the trajectory as well."""
    inst, meta = orc.load_golden(os.path.join(GOLDEN_DIR, name + ".npz"))
    dt = np.float64 if precision == "f64" else np.float32
    L = layout_from_instance(inst)
    eng = HostMgm2(L, precision=precision, mode=meta["mode"], seed=meta["seed"], var_rank=inst["var_rank"],
                   **meta["params"]).init()
    if precision == "f64" or "float" not in name:
        check_trajectory(eng, inst, meta, dt, name)
        return
    o = Mgm2Oracle(inst, dt, mode=meta["mode"], seed=meta["seed"], **meta["params"]).init()
    for k in range(meta["n_cycles"] + 1):
        if k:
            o.step()
            eng.step()
            _assert_same(eng.record(), o.record(), dt, k)
        assert np.array_equal(eng.values()[0], o.values()[0]), k
        assert np.array_equal(eng.values()[1].astype(dt), o.values()[1].astype(dt), equal_nan=True), k


def random_mgm2_instance(n, d, arities, seed, n_factors=None, levels=0):
    """Mixed-arity random graph with float tables (or integer costs in [0, levels): ties, so `favor`
    decides), random name ranks and some initial values."""
    rng = np.random.default_rng(seed)
    parts = []
    for i, a in enumerate(arities):
        nf = n_factors or (n if a > 1 else n // 10)
        parts.append(random_factor_graph(n, d, nf, a, seed=seed + i, noise=0.5, int_tables=False))
    inst = dict(parts[0])
    fp, ev, tb = [parts[0]["factor_ptr"]], [parts[0]["edge_var"]], [parts[0]["tables"]]
    for p in parts[1:]:
        fp.append(p["factor_ptr"][1:] + fp[-1][-1])
        ev.append(p["edge_var"])
        tb.append(p["tables"])
    inst["factor_ptr"] = np.concatenate(fp)
    inst["edge_var"] = np.concatenate(ev).astype(np.int32)
    inst["tables"] = np.concatenate(tb)
    if levels:
        inst["tables"] = np.floor(np.abs(inst["tables"]) * 7) % levels
    inst.pop("table_off", None)
    inst["var_rank"] = rng.permutation(n).astype(np.int32)
    inst["init_value"] = np.where(rng.random(n) < 0.3, rng.integers(0, d, n), -1).astype(np.int32)
    inst["var_ptr"], inst["var_edge"] = default_var_csr(n, inst["edge_var"])
    return inst


@pytest.mark.parametrize("precision,mode,favor,threshold,levels", [("f64", "min", "unilateral", 0.5, 0),
                                                                  ("f32", "min", "no", 0.4, 0),
                                                                  ("f32", "max", "coordinated", 0.7, 0),
                                                                  ("f64", "max", "no", 0.5, 0),
                                                                  ("f32", "max", "no", 0.5, 2),
                                                                  ("f64", "min", "no", 0.5, 2),
                                                                  ("f64", "max", "coordinated", 0.5, 3),
                                                                  ("f32", "min", "coordinated", 0.5, 2)])
def test_kernel_source_matches_oracle_on_random_graphs(precision, mode, favor, threshold, levels):
    """Float costs, and integer costs with few levels, where the favor rule decides ties."""
    inst = random_mgm2_instance(600, 4 if not levels else 3, [2, 3, 1], seed=11, levels=levels)
    dt = np.float64 if precision == "f64" else np.float32
    kw = dict(mode=mode, favor=favor, threshold=threshold, seed=5)
    o = Mgm2Oracle(inst, dt, **kw).init()
    eng = HostMgm2(layout_from_instance(inst), precision=precision, var_rank=inst["var_rank"], **kw).init()
    assert np.array_equal(eng.values()[0], o.values()[0])
    pairs = 0
    for k in range(1, 9):
        o.step()
        eng.step()
        rec = o.record()
        _assert_same(eng.record(), rec, dt, k)
        assert np.array_equal(eng.values()[0], o.values()[0]), k
        assert np.array_equal(eng.values()[1].astype(dt), o.values()[1].astype(dt), equal_nan=True), k
        pairs += int(rec["go"].sum())
    assert pairs > 0
    if levels:
        assert o.stats["ties"] > 0
        if favor == "no":
            assert o.stats["coin_commit"] > 0 and o.stats["coin_refuse"] > 0
        else:
            assert o.stats["tie_commits"] == o.stats["ties"]


def test_offer_offsets():
    inst = random_mgm2_instance(200, 3, [2], seed=2)
    inst["dom_size"] = np.where(np.arange(200) % 2 == 0, 3, 5).astype(np.int32)
    ts = [np.prod(inst["dom_size"][inst["edge_var"][inst["factor_ptr"][f]:inst["factor_ptr"][f + 1]]])
          for f in range(len(inst["factor_ptr"]) - 1)]
    inst["tables"] = np.zeros(int(np.sum(ts)))
    inst["unary"] = np.zeros(int(inst["dom_size"].sum()))
    L = layout_from_instance(inst)
    h = mgm_host_arrays(L)
    off, size = mgm2_offer_offsets(L, h["nbr_ptr"], h["nbr_idx"])
    for v in range(L.n_vars):
        nb = h["nbr_idx"][h["nbr_ptr"][v]:h["nbr_ptr"][v + 1]]
        want = int(L.dom_size[v]) * (int(L.dom_size[nb].max()) if len(nb) else 0)
        end = off[v + 1] if v + 1 < L.n_vars else size
        assert end - off[v] == want


def test_descriptor_validation():
    """fg_mgm2_create refuses a bad descriptor with FG_ERR_ARG and a message, and without a device reports
    FG_ERR_CUDA — never a CPU path."""
    import torch
    lib = _cabi.load()
    inst = random_mgm2_instance(60, 3, [2], seed=1)
    d = HostMgm2(layout_from_instance(inst)).d

    def create():
        h = P()
        rc = lib.fg_mgm2_create(C.byref(d), C.byref(h))
        msg = (lib.fg_mgm2_last_error(h) or b"").decode()
        lib.fg_mgm2_destroy(h)
        return rc, msg

    d.favor = 7
    rc, msg = create()
    assert rc == _cabi.FG_ERR_ARG and "favor" in msg
    d.favor, d.threshold = 1, 1.5
    rc, msg = create()
    assert rc == _cabi.FG_ERR_ARG and "threshold" in msg
    d.threshold, offer = 0.5, d.dev_offer
    d.dev_offer = None
    rc, msg = create()
    assert rc == _cabi.FG_ERR_ARG and "missing" in msg
    d.dev_offer = offer
    if not torch.cuda.is_available():
        rc, msg = create()
        assert rc == _cabi.FG_ERR_CUDA and "no CUDA device" in msg


def test_kernel_source_no_neighbors():
    """The reference's test_no_neighbors through the init kernel: max mode, cost x1 * 2 over 0..9 gives
    value 9 with cost 18."""
    from test_mgm2_cpu import unit_instance
    inst = unit_instance([list(range(10))], [([0], lambda x1: x1 * 2)])
    for precision in ("f64", "f32"):
        eng = HostMgm2(layout_from_instance(inst), precision=precision, mode="max").init()
        val, cost = eng.values()
        assert val.tolist() == [9] and cost.tolist() == [18.0]


@pytest.mark.parametrize("precision,mode,favor", [("f32", "min", "no"), ("f64", "max", "coordinated")])
@pytest.mark.parametrize("case", list(LM.LOCAL))
def test_kernel_source_at_the_limits(case, precision, mode, favor):
    """Domain sizes 1 and 256 and the mix {1, 2, 256} (tests/_limits.py), as tests/test_gpu_limits.py runs them."""
    inst = LM.LOCAL[case]()
    dt = np.float64 if precision == "f64" else np.float32
    kw = dict(mode=mode, favor=favor, threshold=0.5, seed=19)
    o = Mgm2Oracle(inst, dt, **kw).init()
    eng = HostMgm2(layout_from_instance(inst), precision=precision, var_rank=inst["var_rank"], **kw).init()
    assert np.array_equal(eng.values()[0], o.values()[0])
    offers = 0
    for k in range(1, 5):
        o.step()
        eng.step()
        rec = o.record()
        _assert_same(eng.record(), rec, dt, k)
        assert np.array_equal(eng.values()[0], o.values()[0]), k
        assert np.array_equal(eng.values()[1].astype(dt), o.values()[1].astype(dt), equal_nan=True), k
        offers += int(rec["offerer"].sum())
    assert offers > 0
