"""GPU: every engine family on a device other than the current one.  A handle belongs to the device current when it
is created (the Python engines make their own device current for every C call) and each C entry point runs on that
device whatever the calling thread has current; every array of a descriptor must live there.

With two devices, an engine on cuda:1 while cuda:0 stays current must equal its oracle bit for bit on every path the
family dispatches to, leave cuda:0 current after every call and keep every tensor on cuda:1; fresh processes check
the per-device launch set-up of the shared-memory kernels whichever device comes first; the C-level device guard
holds without the Python wrapper; solve() gives the same answer on either device; two MaxSum shards on two devices
equal the single-GPU engine.  With one device, each family's create refuses host memory in a descriptor."""
import ctypes as C
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

import _limits as LM
import oracle as orc
from _dba_oracle import DbaOracle
from _dpop_oracle import DpopOracle
from _gdba_oracle import GdbaOracle
from _mgm2_oracle import Mgm2Oracle
from bench import oracle_instance
from conftest import ROOT
from pydcop_b200 import pseudotree as pt
from pydcop_b200.generators import mixed_shape_graph, random_factor_graph
from pydcop_b200.layout import build_layout, layout_from_instance
from test_dba_hostshim import random_dba_instance
from test_gdba_hostshim import compare_with_oracle as compare_gdba
from test_gpu_dsa_cached import _inst as dsa_binary_instance
from test_gpu_fast import _mixed_instance
from test_gpu_limits import _compare_maxsum
from test_gpu_narrow_tables import _int8_instance
from test_gpu_tiled_rt import MIXED
from test_gpu_zz_dba import check_bits, compare_with_oracle as compare_dba, limit_instance
from test_gpu_zz_dpop import _check_engine as check_dpop
from test_mgm2_hostshim import _assert_same as assert_same_mgm2

pytestmark = pytest.mark.gpu

N_DEV = torch.cuda.device_count() if torch.cuda.is_available() else 0
two_devices = pytest.mark.skipif(N_DEV < 2, reason="needs two CUDA devices (cuda:0 and cuda:1)")
DEV1 = "cuda:1"


def _dt(precision):
    return np.float64 if precision == "f64" else np.float32


def _tensors(eng):
    """Every device tensor an engine holds (attributes, lists and dicts of them)."""
    out = []
    for v in vars(eng).values():
        for x in (v if isinstance(v, (list, tuple)) else v.values() if isinstance(v, dict) else [v]):
            if isinstance(x, torch.Tensor):
                out.append(x)
    return out


def _on_dev1(eng):
    """cuda:0 is still current and every tensor of the engine lives on cuda:1."""
    assert torch.cuda.current_device() == 0
    assert eng.device == torch.device(DEV1)
    ts = _tensors(eng)
    assert ts and all(t.device == torch.device(DEV1) for t in ts), {t.device for t in ts}


@pytest.fixture
def dev0_current():
    """cuda:0 current for the test, whatever ran before."""
    prev = torch.cuda.current_device()
    torch.cuda.set_device(0)
    yield
    torch.cuda.set_device(prev)


# ---------------------------------------------------------------------------------------------------------------
# 1. every family on cuda:1 while cuda:0 stays current
def _maxsum_on_dev1(inst, precision, cycles, **params):
    from pydcop_b200 import MaxSumEngine
    L = build_layout(**inst)
    o = orc.MaxSumOracle(oracle_instance(inst, L), _dt(precision), **params).init()
    eng = MaxSumEngine(L, device=DEV1, precision=precision, **params)
    _on_dev1(eng)
    eng.init()
    _on_dev1(eng)
    for k in range(cycles):
        if k:
            o.step()
            eng.step()
            _on_dev1(eng)
        _compare_maxsum(eng, o, k)
    _on_dev1(eng)
    return L, eng


def _hub_instance():
    inst = random_factor_graph(400, 4, 900, 2, seed=9)
    inst["edge_var"] = inst["edge_var"].copy()
    inst["edge_var"][0:400:2] = 7          # variable 7 becomes a hub of degree ~200
    ev = inst["edge_var"].reshape(-1, 2)
    ev[ev[:, 0] == ev[:, 1], 1] = 8        # keep scopes distinct
    return inst


MAXSUM_PATHS = {
    "warp_int8_d10": (lambda: _int8_instance(10, seed=70), "f32"),
    "warp_float": (lambda: random_factor_graph(900, 10, 1900, 2, seed=71, int_tables=False), "f32"),
    "pipe_arity3": (lambda: _mixed_instance(600, 4, 700, 3, n_unary=200, seed=72), "f32"),
    "tiled_rt_mixed": (lambda: mixed_shape_graph(seed=3, **MIXED), "f64"),
    "generic_hub": (_hub_instance, "f32"),
}


@two_devices
@pytest.mark.parametrize("path", list(MAXSUM_PATHS))
def test_maxsum_on_second_device(path, dev0_current):
    build, precision = MAXSUM_PATHS[path]
    inst = build()
    L, eng = _maxsum_on_dev1(inst, precision, 8)
    fam, widths = eng.kernel_plan(), eng.table_widths()
    _on_dev1(eng)
    full = np.dtype(_dt(precision)).itemsize
    if path == "warp_int8_d10":
        assert "warp" in fam and {w for w, f in zip(widths, fam) if f == "warp"} == {1}
    elif path == "warp_float":
        assert "warp" in fam and {w for w, f in zip(widths, fam) if f == "warp"} == {full}
    elif path == "pipe_arity3":
        assert any(c.arity == 3 and f == "pipe" for c, f in zip(L.classes, fam)), fam
    elif path == "tiled_rt_mixed":
        assert "tiled_rt" in fam
    else:
        # variables of degree > 16 share the irregular class (degree -1), which no tiled variable-side kernel takes
        # (maxsum_fast_plan): k_v2f_generic alone writes their q rows.  The hub's rows were written on cuda:1 (they
        # start at zero and the hub posts nothing at start) and equal the oracle's (_compare_maxsum above).
        assert any(vc.degree == -1 and vc.n_slots > 0 for vc in L.var_classes)
        ev = np.asarray(inst["edge_var"])
        assert (ev == 7).sum() > 32
        off = np.concatenate([[0], np.cumsum(np.asarray(inst["dom_size"])[ev])])
        q = eng.messages()[0]
        rows = [q[off[e]:off[e + 1]] for e in np.flatnonzero(ev == 7)]
        assert all(np.any(r != 0) for r in rows)
    eng.close()
    assert torch.cuda.current_device() == 0


def _dsa_on_dev1(inst, precision, cycles, **kw):
    from pydcop_b200 import DsaEngine
    L = build_layout(**inst)
    o = orc.DsaOracle(oracle_instance(inst, L), _dt(precision), **kw).init()
    eng = DsaEngine(L, device=DEV1, precision=precision, **kw).init()
    _on_dev1(eng)
    assert np.array_equal(eng.values(), o.val)
    for k in range(1, cycles + 1):
        o.step()
        eng.step()
        _on_dev1(eng)
        assert np.array_equal(eng.values(), o.val), k
        assert eng.cycle == k
    _on_dev1(eng)
    return eng


@two_devices
@pytest.mark.parametrize("path", ["cached", "generic", "adsa"])
def test_dsa_on_second_device(path, dev0_current):
    if path == "cached":
        eng = _dsa_on_dev1(dsa_binary_instance(6000, 20, 17000, seed=23), "f32", 12, mode="min", variant="B", seed=5)
        assert eng.row_cache is not None
    elif path == "generic":
        eng = _dsa_on_dev1(LM.DSA["hub2400"](), "f64", 10, mode="max", variant="A", seed=7, probability=0.7)
        assert eng.tables_or is None and eng.row_cache is None
    else:
        rng = np.random.default_rng(5)
        inst = random_factor_graph(3000, 10, 8000, 2, seed=30, noise=0.0)
        inst["tables"] = rng.integers(0, 3, len(inst["tables"])).astype(np.float32)
        inst["unary"] = np.round(rng.uniform(0, 2, len(inst["unary"])), 2)
        eng = _dsa_on_dev1(inst, "f64", 10, mode="max", variant="A", seed=9, var_costs=True)
        assert eng.tables_or is not None
    eng.close()
    assert torch.cuda.current_device() == 0


MGM_PATHS = {
    "cached_d10_f32": (lambda: LM.mgm_hub(10), "f32", "max"),
    "cached_d20": (lambda: LM.mgm_hub(20), "f64", "min"),
    "generic_d1": (lambda: LM.MGM["d1"](), "f32", "min"),
}


@two_devices
@pytest.mark.parametrize("path", list(MGM_PATHS))
def test_mgm_on_second_device(path, dev0_current):
    from pydcop_b200.engine import MgmEngine
    build, precision, mode = MGM_PATHS[path]
    inst = build()
    dt = _dt(precision)
    o = orc.MgmOracle(inst, dt, mode=mode, seed=17).init()
    eng = MgmEngine(layout_from_instance(inst), device=DEV1, precision=precision, mode=mode, seed=17,
                    var_rank=inst["var_rank"]).init()
    _on_dev1(eng)
    assert np.array_equal(eng.values()[0], o.val)
    for k in range(1, 9):
        o.step()
        eng.step()
        _on_dev1(eng)
        val, cost = eng.values()
        assert np.array_equal(val, o.val), k
        assert np.array_equal(cost.astype(dt), o.cost, equal_nan=True), k
        gain, new_value = eng.gains()
        assert np.array_equal(gain.astype(dt), o.gain) and np.array_equal(new_value, o.new_val), k
        assert eng.cycle == k
    if path.startswith("cached"):
        assert eng.fast_chunk in (2, 4) and eng.row_cache is not None
    else:
        assert eng.fast_chunk == 0
    _on_dev1(eng)
    eng.close()


@two_devices
def test_mgm2_on_second_device(dev0_current):
    from pydcop_b200.engine import Mgm2Engine
    inst = LM.LOCAL["doms_1_2_256"]()
    dt = np.float64
    kw = dict(mode="max", favor="coordinated", threshold=0.5, seed=19)
    o = Mgm2Oracle(inst, dt, **kw).init()
    eng = Mgm2Engine(layout_from_instance(inst), device=DEV1, precision="f64", var_rank=inst["var_rank"], **kw).init()
    _on_dev1(eng)
    assert np.array_equal(eng.values()[0], o.values()[0])
    pairs = 0
    for k in range(1, 5):
        o.step()
        eng.step()
        _on_dev1(eng)
        rec = o.record()
        assert_same_mgm2(eng.record(), rec, dt, k)
        assert np.array_equal(eng.values()[0], o.values()[0]), k
        assert eng.cycle == k
        pairs += int(rec["go"].sum())
    assert pairs > 0
    _on_dev1(eng)
    eng.close()


@two_devices
def test_gdba_on_second_device(dev0_current):
    from pydcop_b200.engine import GdbaEngine
    inst = LM.gdba_instance("doms_1_2_256")
    kw = dict(mode="min", modifier="M", violation="NZ", increase_mode="R", seed=23)
    o = GdbaOracle(inst, np.float32, **kw).init()
    eng = GdbaEngine(layout_from_instance(inst), device=DEV1, precision="f32", var_rank=inst["var_rank"], **kw).init()
    _on_dev1(eng)
    compare_gdba(eng, o, np.float32, 6)
    assert eng.cycle == 6 and o.stats["breakouts"] > 0
    _on_dev1(eng)
    eng.close()


@two_devices
@pytest.mark.parametrize("dmax", [32, 256])
def test_dba_on_second_device(dmax, dev0_current):
    from pydcop_b200.engine import DbaEngine
    if dmax == 32:
        inst, precision, infinity, max_distance, n = random_dba_instance(5000, 3, seed=17), "f64", 10000, 2, 14
    else:
        inst, precision, infinity, max_distance, n = limit_instance("d256"), "f32", 10000, 3, 5
    assert (int(inst["dom_size"].max()) <= 32) == (dmax == 32)
    kw = dict(infinity=infinity, max_distance=max_distance, seed=29)
    o = DbaOracle(inst, _dt(precision), **kw).init()
    eng = DbaEngine(layout_from_instance(inst), device=DEV1, precision=precision, var_rank=inst.get("var_rank"),
                    **kw).init()
    _on_dev1(eng)
    check_bits(eng, precision, infinity)
    compare_dba(eng, o, n)       # also reads cycle / finished (fg_dba_current) after every round
    _on_dev1(eng)
    eng.close()


@two_devices
@pytest.mark.parametrize("case", ["d256_big_nodes", "walk_domain_one"])
def test_dpop_on_second_device(case, dev0_current):
    from pydcop_b200.engine import DpopEngine
    inst = LM.dpop_d256() if case == "d256_big_nodes" else LM.dpop_with_domain_one()
    t = pt.build_tree(inst["dom_size"], inst["factor_ptr"], inst["edge_var"])
    L = build_layout(inst["dom_size"], inst["factor_ptr"], inst["edge_var"], inst["tables"], unary=inst["unary"])
    eng = DpopEngine(L, t, device=DEV1, precision="f64", mode="min").init()
    _on_dev1(eng)
    eng.step()
    _on_dev1(eng)
    assert eng.finished and eng.launch_count == eng.sched.n_launches
    assert bool(eng.sched.big_nodes) == (case == "d256_big_nodes")
    o = DpopOracle(inst, t, np.float64, "min").run()
    check_dpop(eng, t, lambda u: o.util[u], o.value, o.cost, np.float64)
    assert eng.unresolved == o.unresolved == 0
    _on_dev1(eng)
    eng.close()


# ---------------------------------------------------------------------------------------------------------------
# 2. fresh processes: the same two engines first on one device, then on the other, all four alive and stepped in
# turn.  The launch code of a kernel instantiation that takes more than the default 48 KB of dynamic shared memory
# sets the attribute once per device; built on one device only, the second device's launch fails.  Both engines
# reach such an instantiation on both devices: every launch of the runtime-shape kernel takes FG_TILED_RT_SMEM or
# FG_TILED_RT_SMEM_BIG bytes, and the f64 d = 8 variable-side warp kernel 4 x 12 KB of stages plus its barriers.
_FRESH = textwrap.dedent("""
    import sys
    sys.path[:0] = [{root!r}, {oracle!r}, {tests!r}]
    import numpy as np
    import torch
    import oracle as orc
    from bench import oracle_instance
    from pydcop_b200 import MaxSumEngine, build_layout
    from pydcop_b200.generators import mixed_shape_graph, random_factor_graph
    from test_gpu_limits import _compare_maxsum
    from test_gpu_tiled_rt import MIXED
    torch.cuda.set_device(0)
    insts = {{"warp": random_factor_graph(900, 8, 1900, 2, seed=92, int_tables=False),
              "tiled_rt": mixed_shape_graph(seed=3, **MIXED)}}
    runs = []
    for dev in ({first!r}, {second!r}):
        for path, inst in insts.items():
            L = build_layout(**inst)
            eng = MaxSumEngine(L, device=dev, precision="f64").init()
            assert path in eng.kernel_plan(), (path, eng.kernel_plan())
            runs.append((eng, orc.MaxSumOracle(oracle_instance(inst, L), np.float64).init()))
    for k in range(1, 7):
        for eng, o in runs:                  # every engine alive, stepped in turn
            eng.step()
            o.step()
            _compare_maxsum(eng, o, k)
            assert torch.cuda.current_device() == 0
    print("ok", [str(e.device) for e, _ in runs])
""")


def _tiled_rt_smem():
    """The dynamic shared memory of the runtime-shape kernel's two launch groups, from its source."""
    import re
    src = open(os.path.join(ROOT, "pydcop_b200", "csrc", "maxsum_tiled_rt.cuh")).read()
    return [int(eval(re.search(r"constexpr size_t %s = ([0-9 *]+);" % name, src).group(1)))
            for name in ("FG_TILED_RT_SMEM", "FG_TILED_RT_SMEM_BIG")]


def test_runtime_shape_kernel_needs_the_shared_memory_attribute():
    """What makes the fresh-process test below meaningful: every launch of k_f2v_tiled_rt is above the 48 KB a
    kernel may take without cudaFuncAttributeMaxDynamicSharedMemorySize."""
    assert min(_tiled_rt_smem()) > 48 * 1024


@two_devices
@pytest.mark.parametrize("first,second", [("cuda:1", "cuda:0"), ("cuda:0", "cuda:1")])
def test_warp_engines_in_a_fresh_process(first, second):
    code = _FRESH.format(root=ROOT, oracle=os.path.join(ROOT, "oracle"), tests=os.path.join(ROOT, "tests"),
                         first=first, second=second)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    assert r.stdout.strip().endswith(str([first, first, second, second])), r.stdout


# ---------------------------------------------------------------------------------------------------------------
# 3. the C-level guard on its own: a cuda:0 handle stepped through raw ctypes while cuda:1 is current
@two_devices
def test_c_entry_points_switch_to_the_handle_device(dev0_current):
    from pydcop_b200 import MaxSumEngine
    inst = _int8_instance(10, seed=93)
    L = build_layout(**inst)
    o = orc.MaxSumOracle(oracle_instance(inst, L), np.float32).init()
    eng = MaxSumEngine(L, device="cuda:0", precision="f32")
    lib, h = eng.lib, eng._h
    st = C.c_void_p(torch.cuda.current_stream(0).cuda_stream)
    torch.cuda.set_device(1)
    try:
        assert lib.fg_maxsum_init(h, st) == 0
        assert torch.cuda.current_device() == 1
        assert lib.fg_maxsum_step(h, 3, st) == 0
        assert torch.cuda.current_device() == 1
        for _ in range(2):
            assert lib.fg_maxsum_cycle_compute(h, st) == 0 and lib.fg_maxsum_cycle_commit(h) == 0
        assert torch.cuda.current_device() == 1
        buf, cyc = C.c_int32(), C.c_int64()
        assert lib.fg_maxsum_current(h, C.byref(buf), C.byref(cyc)) == 0 and cyc.value == 5
        out = (C.c_int32 * len(L.classes))()
        assert lib.fg_maxsum_kernel_plan(h, out, len(L.classes)) == 0 and 2 in list(out)   # FG_KERNEL_WARP
        assert torch.cuda.current_device() == 1
        torch.cuda.synchronize(0)
    finally:
        torch.cuda.set_device(0)
    o.step(5)
    _compare_maxsum(eng, o, 5)
    # the same handle closed with cuda:1 current: the destroy runs on cuda:0 too
    torch.cuda.set_device(1)
    try:
        assert lib.fg_maxsum_destroy(h) == 0
        eng._h = C.c_void_p()
        assert torch.cuda.current_device() == 1
    finally:
        torch.cuda.set_device(0)


@two_devices
def test_create_refuses_arrays_of_another_device(dev0_current):
    """A descriptor whose arrays live on cuda:1, created with cuda:0 current: FG_ERR_ARG naming both devices."""
    from pydcop_b200 import MaxSumEngine, _cabi
    L = build_layout(**_int8_instance(10, seed=94))
    eng = MaxSumEngine(L, device=DEV1, precision="f32")
    h = C.c_void_p()
    rc = eng.lib.fg_maxsum_create(C.byref(eng._desc), C.byref(h))
    msg = (eng.lib.fg_maxsum_last_error(h) or b"").decode()
    eng.lib.fg_maxsum_destroy(h)
    assert rc == _cabi.FG_ERR_ARG and msg == "dev_tables is device memory of device 1, the handle belongs to device 0"
    assert torch.cuda.current_device() == 0


# ---------------------------------------------------------------------------------------------------------------
# 4. solve() on either device
SOLVE_PARAMS = {"maxsum": {"stop_cycle": 12}, "dsa": {"stop_cycle": 15}, "adsa": {"stop_cycle": 15},
                "mgm": {"stop_cycle": 15}, "mgm2": {"stop_cycle": 10}, "gdba": {"stop_cycle": 15},
                "dba": {"stop_cycle": 30}, "dpop": {}}


@two_devices
@pytest.mark.parametrize("algo", list(SOLVE_PARAMS))
def test_solve_gives_the_same_answer_on_either_device(algo, dev0_current):
    from pydcop_b200 import solve as S
    inst = LM.dpop_with_domain_one()
    arrays = {k: np.asarray(inst[k]) for k in ("dom_size", "factor_ptr", "edge_var", "tables", "unary")}
    res = [S.solve(arrays, algo, SOLVE_PARAMS[algo], precision="f64", seed=3, device=dev) for dev in ("cuda:0", DEV1)]
    assert torch.cuda.current_device() == 0
    for key in ("assignment", "cost", "violation", "cycle", "status"):
        assert res[0][key] == res[1][key], key
    assert res[0]["cycle"] == (0 if algo == "dpop" else SOLVE_PARAMS[algo]["stop_cycle"]) or algo == "dba"


# ---------------------------------------------------------------------------------------------------------------
# 5. two MaxSum shards of one process on two devices
class _CrossDeviceFabric:
    """all_to_all_single between in-process shards on different devices: each block is copied to the receiver's
    device."""

    def __init__(self, shards):
        self.shards = shards

    def exchange(self):
        for s in self.shards:
            torch.cuda.synchronize(s.device)
        for a, sa in enumerate(self.shards):
            so = np.concatenate([[0], np.cumsum(sa.halo.send_split)]).astype(int)
            for b, sb in enumerate(self.shards):
                ro = np.concatenate([[0], np.cumsum(sb.halo.recv_split)]).astype(int)
                n = so[b + 1] - so[b]
                assert n == ro[a + 1] - ro[a]
                if n:
                    sb.halo.buf_recv[ro[a]:ro[a + 1]] = sa.halo.buf_send[so[b]:so[b + 1]].to(sb.device)
        for s in self.shards:
            torch.cuda.synchronize(s.device)


def _run_two_device_shards(inst, cycles):
    from pydcop_b200.multigpu import ShardedMaxSum
    shards = [ShardedMaxSum(inst, r, 2, f"cuda:{r}", precision="f32") for r in range(2)]
    assert [s.device for s in shards] == [torch.device("cuda:0"), torch.device(DEV1)]
    fab = _CrossDeviceFabric(shards)

    def halo(bufsel):
        for s in shards:
            s.halo.pack_rows(*bufsel(s.engine))
        fab.exchange()
        for s in shards:
            s.halo.unpack_rows(*bufsel(s.engine))

    for s in shards:
        s.engine.init()
    halo(lambda e: (e.q[0], e.r[0]))
    for name_send, name_recv, rows, rs in (("send_r_edge", "recv_r_edge", "r_valid", "send_r_rows"),
                                           ("send_q_edge", "recv_q_edge", "q_valid", "send_q_rows")):
        outs = [getattr(s.engine, rows)[torch.from_numpy(getattr(s.plan, name_send).astype(np.int64)).to(s.device)]
                for s in shards]
        for b, sb in enumerate(shards):
            parts = []
            for a, sa in enumerate(shards):
                so = np.concatenate([[0], np.cumsum(getattr(sa.plan, rs))]).astype(int)
                parts.append(outs[a][so[b]:so[b + 1]].to(sb.device))
            idx = torch.from_numpy(getattr(sb.plan, name_recv).astype(np.int64)).to(sb.device)
            if len(idx):
                getattr(sb.engine, rows)[idx] = torch.cat(parts)
    for _ in range(cycles):
        for s in shards:
            s.engine.cycle_compute()
        halo(lambda e: (e.q[e.cur ^ 1], e.r[e.cur ^ 1]))
        for s in shards:
            s.engine.cycle_commit()
        assert torch.cuda.current_device() == 0
    for s in shards:
        torch.cuda.synchronize(s.device)
    return shards


@two_devices
@pytest.mark.parametrize("kind", ["uniform_d10", "mixed_arity"])
def test_two_shards_on_two_devices_equal_single_gpu(kind, dev0_current):
    from pydcop_b200 import MaxSumEngine
    if kind == "uniform_d10":
        inst = random_factor_graph(1500, 10, 3000, 2, seed=2)
    else:
        inst = random_factor_graph(600, 4, 900, 2, seed=3)
        t = random_factor_graph(600, 4, 200, 3, seed=4)
        inst["edge_var"] = np.concatenate([inst["edge_var"], t["edge_var"]])
        inst["factor_ptr"] = np.concatenate([inst["factor_ptr"], inst["factor_ptr"][-1] + t["factor_ptr"][1:]])
        inst["tables"] = np.concatenate([inst["tables"], t["tables"]])
    cycles = 9
    L = build_layout(**inst)
    ref = MaxSumEngine(L, device="cuda:0", precision="f32").init().step(cycles)
    ref_q, ref_r = ref.messages()
    ref_val = ref.values()[0]
    shards = _run_two_device_shards(inst, cycles)
    dom = inst["dom_size"][inst["edge_var"]]
    off = np.concatenate([[0], np.cumsum(dom)])
    val = np.full(len(inst["dom_size"]), -1)
    for s in shards:
        ids, v = s.local_values()
        val[ids] = v
        q, r = s.engine.messages()
        Ls = s.plan.layout
        loff = np.concatenate([[0], np.cumsum(Ls.canon_dom_size[Ls.canon_edge_var])])
        canon = np.concatenate([s.plan.own_factor_edges, s.plan.stub_edges])
        for le, ge in enumerate(canon):
            d = int(dom[ge])
            assert np.array_equal(r[loff[le]:loff[le] + d], ref_r[off[ge]:off[ge] + d]), ("r", ge)
            assert np.array_equal(q[loff[le]:loff[le] + d], ref_q[off[ge]:off[ge] + d]), ("q", ge)
    assert np.array_equal(val, ref_val)
    assert all(len(s.plan.send_r_edge) for s in shards)     # the cut is not empty


# ---------------------------------------------------------------------------------------------------------------
# 6. one device: every family's create refuses a descriptor array in host memory before any device work
def _family_engines():
    from pydcop_b200.engine import DbaEngine, DpopEngine, DsaEngine, GdbaEngine, MaxSumEngine, Mgm2Engine, MgmEngine
    inst = LM.with_local_search_arrays(LM.random_graph(200, [3], [(2, 300), (1, 20)], seed=95, levels=3), 5)
    L = layout_from_instance(inst)
    tree_inst = LM.dpop_with_domain_one()          # separators of a few variables: DPOP's UTIL tables stay small
    t = pt.build_tree(tree_inst["dom_size"], tree_inst["factor_ptr"], tree_inst["edge_var"])
    Lt = build_layout(tree_inst["dom_size"], tree_inst["factor_ptr"], tree_inst["edge_var"], tree_inst["tables"],
                      unary=tree_inst["unary"])
    return {
        "maxsum": lambda: MaxSumEngine(L, precision="f32"),
        "dsa": lambda: DsaEngine(L, precision="f32"),
        "mgm": lambda: MgmEngine(L, precision="f32", var_rank=inst["var_rank"]),
        "mgm2": lambda: Mgm2Engine(L, precision="f32", var_rank=inst["var_rank"]),
        "gdba": lambda: GdbaEngine(L, precision="f32", var_rank=inst["var_rank"]),
        "dba": lambda: DbaEngine(L, precision="f32", var_rank=inst["var_rank"]),
        "dpop": lambda: DpopEngine(Lt, t, precision="f32"),
    }


@pytest.mark.parametrize("memory", ["pinned", "pageable"])
@pytest.mark.parametrize("family", ["maxsum", "dsa", "mgm", "mgm2", "gdba", "dba", "dpop"])
@pytest.mark.parametrize("field", ["dev_tables", "dev_value"])
def test_create_refuses_host_memory(family, memory, field):
    from pydcop_b200 import _cabi
    eng = _family_engines()[family]()
    d = type(eng._desc).from_buffer_copy(eng._desc)
    pair = isinstance(getattr(d, field), C.Array)      # a double buffer: its first half
    target = field + "[0]" if pair else field
    n = 1 << 16
    if memory == "pinned":
        host = torch.full((n,), 7, dtype=torch.uint8, pin_memory=True)
        addr = host.data_ptr()
    else:
        host = np.full(n, 7, dtype=np.uint8)
        addr = host.ctypes.data
    if pair:
        getattr(d, field)[0] = addr
    else:
        setattr(d, field, addr)
    lib = eng.lib
    fn = lambda name: getattr(lib, f"fg_{family}_{name}")  # noqa: E731
    h = C.c_void_p()
    torch.cuda.synchronize()
    rc = fn("create")(C.byref(d), C.byref(h))
    msg = (fn("last_error")(h) or b"").decode()
    fn("destroy")(h)
    torch.cuda.synchronize()
    kind = "pinned host memory" if memory == "pinned" else "pageable host memory"
    dev = eng.device.index
    assert rc == _cabi.FG_ERR_ARG, (rc, msg)
    assert msg == f"{target} is {kind}, not device memory of the handle's device {dev}", msg
    # the residency check is the first device work of create, before any allocation or launch; what a test can see
    # of that is that the host buffer was not written
    assert (np.asarray(host.numpy() if memory == "pinned" else host) == 7).all()
    # the engine's own handle, over the untouched descriptor, still works
    eng.init().step(2)
    torch.cuda.synchronize()
    eng.close()
