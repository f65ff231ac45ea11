"""GPU: the runtime-dimension tiled factor kernel (csrc/maxsum_tiled_rt.cuh) — the shapes the
compile-time kernels do not cover: mixed domain sizes inside a factor, domain sizes outside the
compiled set, arity 4..6 — against the CPU oracle, bit for bit, both precisions, and against the
one-thread-per-edge generic kernel it replaces."""
import numpy as np
import pytest

from pydcop_b200.generators import mixed_shape_graph, random_factor_graph
from test_gpu_fast import _run_pair

pytestmark = pytest.mark.gpu

MIXED = dict(n_vars=700, doms=(2, 3, 5, 7), shapes=[(1, 200), (2, 900), (3, 300), (4, 90)])


@pytest.mark.parametrize("precision", ["f32", "f64"])
def test_mixed_domains_and_arities_bit_exact_vs_oracle(precision):
    inst = mixed_shape_graph(seed=3, **MIXED)
    eng = _run_pair(inst, precision, 9)
    fam = eng.kernel_plan()
    mixed = [f for c, f in zip(eng.layout.classes, fam) if len(set(c.dom[:c.arity])) > 1 or c.arity >= 4]
    assert mixed and all(f == "tiled_rt" for f in mixed), fam
    assert "generic" not in fam


UNIFORM_RT = [(2, 7), (2, 12), (2, 31), (3, 6), (3, 11), (4, 4), (5, 3), (6, 2)]


@pytest.mark.parametrize("arity,d", UNIFORM_RT)
def test_uniform_shapes_outside_the_compiled_set(arity, d):
    n_f = 400
    inst = random_factor_graph(max(120, n_f * arity // 4), d, n_f, arity, seed=40 + arity * d, int_tables=False)
    eng = _run_pair(inst, "f32", 6)
    assert set(eng.kernel_plan()) == {"tiled_rt"}


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("mode", ["min", "max"])
def test_mixed_domains_with_hard_constraints(mode, precision):
    """+/-inf cells and variables with every value forbidden, on the mixed-shape classes"""
    inst = mixed_shape_graph(seed=3, **MIXED)
    eng = _run_pair(inst, precision, 12, hard_sites={"tiled_rt"}, mode=mode)
    assert "tiled_rt" in eng.kernel_plan() and "generic" not in eng.kernel_plan()


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("arity,d", UNIFORM_RT + [(7, 2), (8, 2)])
def test_uniform_shapes_outside_the_compiled_set_with_hard_constraints(arity, d, precision):
    n_f = 400
    inst = random_factor_graph(max(120, n_f * arity // 4), d, n_f, arity, seed=40 + arity * d, int_tables=False)
    mode = "max" if (arity + d) % 2 else "min"
    eng = _run_pair(inst, precision, 12, hard_sites={"tiled_rt"}, mode=mode)
    fam = eng.kernel_plan()
    assert [f for c, f in zip(eng.layout.classes, fam) if c.arity >= 2] == ["tiled_rt"], fam


@pytest.mark.parametrize("params", [
    dict(mode="max"), dict(damping_nodes="none"), dict(damping_nodes="factors", damping=0.3),
    dict(damping_nodes="vars", damping=0.8), dict(stability=0.6), dict(start_messages="all"),
    dict(start_messages="leafs_vars", mode="max", damping=0.25)])
def test_parameter_sweep(params):
    inst = mixed_shape_graph(seed=8, **MIXED)
    _run_pair(inst, "f32", 11, **params)


def test_large_tables():
    """one table per CTA: 54 KB (f32, 72 KB launch), 108 KB (f64, 200 KB launch), and tables that do not fit
    shared memory at all and are read in place (arity 4 over 16 values: 256 KB in f32)"""
    inst = random_factor_graph(60, 24, 40, 3, seed=2, int_tables=False)     # 13 824 entries
    for prec in ("f32", "f64"):
        eng = _run_pair(inst, prec, 4)
        assert set(eng.kernel_plan()) == {"tiled_rt"}
    inst = random_factor_graph(40, 16, 12, 4, seed=6, int_tables=False)     # 65 536 entries
    eng = _run_pair(inst, "f32", 3)
    assert set(eng.kernel_plan()) == {"tiled_rt"}
    inst = mixed_shape_graph(50, (12, 33), [(4, 10), (2, 40)], seed=4)      # last dimension wider than a warp
    eng = _run_pair(inst, "f32", 3)
    assert "generic" not in eng.kernel_plan()


def test_tiled_rt_and_generic_agree(monkeypatch):
    from pydcop_b200 import MaxSumEngine, build_layout
    inst = mixed_shape_graph(seed=5, int_tables=True, **MIXED)
    L = build_layout(**inst)
    a = MaxSumEngine(L, precision="f32").init().step(15)
    monkeypatch.setenv("PYDCOP_B200_TILED_RT", "0")
    b = MaxSumEngine(build_layout(**inst), precision="f32").init().step(15)
    assert "tiled_rt" in a.kernel_plan() and "tiled_rt" not in b.kernel_plan() and "generic" in b.kernel_plan()
    for x, y in zip(a.messages(), b.messages()):
        assert np.array_equal(x, y)
    assert np.array_equal(a.values()[0], b.values()[0])
    assert a.launch_count < b.launch_count      # one launch per arity instead of one per class
