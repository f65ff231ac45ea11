"""GPU: the shape-specialised (tiled, TMA / cp.async staged) kernels against the CPU oracle on
instances large enough to contain full tiles, for every compiled (arity, domain) shape, both
precisions; plus the division-free approx_match against the literal form on adversarial inputs."""
import os

import numpy as np
import pytest

import oracle as orc
from _hard_constraints import forbid, output_site, sites_reached
from bench import oracle_instance
from pydcop_b200.generators import random_factor_graph

pytestmark = pytest.mark.gpu


def _mixed_instance(n_vars, d, n_factors, arity, n_unary, seed):
    inst = random_factor_graph(n_vars, d, n_factors, arity, seed=seed, int_tables=False)
    if n_unary:
        rng = np.random.default_rng(seed + 1)
        uv = rng.integers(0, n_vars, n_unary).astype(np.int32)
        inst["edge_var"] = np.concatenate([inst["edge_var"], uv])
        inst["factor_ptr"] = np.concatenate(
            [inst["factor_ptr"], inst["factor_ptr"][-1] + np.arange(1, n_unary + 1)])
        inst["tables"] = np.concatenate(
            [inst["tables"], rng.uniform(0, 3, n_unary * d).astype(np.float32)])
    return inst


def _run_pair(inst, precision, cycles, hard_sites=None, **params):
    """Engine against the same-precision oracle after `cycles` cycles, bit for bit (NaN where the oracle
    has NaN).  hard_sites: forbid assignments first (tests/_hard_constraints.py::forbid, +inf cells in min
    mode, -inf in max mode, and variables with every value forbidden) and require that the oracle meets an
    output with only NaN candidates on one of these sites (output_site names)."""
    from pydcop_b200 import MaxSumEngine, build_layout
    if hard_sites is not None:
        inst = forbid(inst, -1.0 if params.get("mode") == "max" else 1.0, seed=len(inst["tables"]))
    L = build_layout(**inst)
    npdt = np.float64 if precision == "f64" else np.float32
    oinst = oracle_instance(inst, L)
    o = orc.MaxSumOracle(oinst, npdt, **params).init()
    reached = set()
    for _ in range(cycles):
        if hard_sites is not None and not (reached & hard_sites):
            reached |= sites_reached(oinst, o.q, o.q_flags & 1)
        o.step()
    if hard_sites is not None:
        assert reached & hard_sites, ("no all-NaN marginal on", hard_sites, reached)
    eng = MaxSumEngine(L, precision=precision, **params).init().step(cycles)
    q, r = eng.messages()
    val, cost = eng.values()
    fl = eng.flags()
    assert np.array_equal(q, o.q.astype(np.float64), equal_nan=True), "q"
    assert np.array_equal(r, o.r.astype(np.float64), equal_nan=True), "r"
    assert np.array_equal(val, o.value), "value"
    assert np.array_equal(cost, o.value_cost.astype(np.float64), equal_nan=True), "value_cost"
    assert np.array_equal(fl["q_sent"], o.q_sent) and np.array_equal(fl["r_sent"], o.r_sent)
    assert np.array_equal(fl["r_cnt"] >> 1, o.r_flags >> 2), "r count"
    assert np.array_equal(fl["q_cnt"] >> 1, o.q_flags >> 2), "q count"
    return eng


SHAPES = [(2, d) for d in (2, 3, 4, 5, 6, 8, 10, 16, 20)] + [(3, d) for d in (2, 3, 4, 5, 8)]


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("arity,d", SHAPES)
def test_tiled_kernels_bit_exact_vs_oracle(arity, d, precision):
    n_factors = 1500 if d <= 4 else 700
    n_vars = max(300, (n_factors * arity) // 4)
    inst = _mixed_instance(n_vars, d, n_factors, arity, n_unary=600, seed=100 + 7 * d + arity)
    _run_pair(inst, precision, 8)


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("arity,d", SHAPES)
def test_tiled_kernels_with_hard_constraints(arity, d, precision):
    """+/-inf cells and variables with every value forbidden: inf and NaN messages, and position-0
    marginals whose candidates are all NaN (the reference keeps +/-inf there)."""
    n_factors = 1500 if d <= 4 else 700
    n_vars = max(300, (n_factors * arity) // 4)
    inst = _mixed_instance(n_vars, d, n_factors, arity, n_unary=600, seed=100 + 7 * d + arity)
    mode = "max" if SHAPES.index((arity, d)) % 2 else "min"
    _run_pair(inst, precision, 12, hard_sites={output_site((d,) * arity, 0, x) for x in range(d)}, mode=mode)


@pytest.mark.parametrize("params", [
    dict(mode="max"), dict(damping_nodes="none"), dict(damping_nodes="vars", damping=0.7),
    dict(damping_nodes="factors", damping=0.2), dict(stability=0.5), dict(stability=1e-4),
    dict(start_messages="all"), dict(start_messages="leafs_vars")])
def test_tiled_kernels_parameter_sweep(params):
    inst = _mixed_instance(900, 10, 1800, 2, n_unary=300, seed=5)
    _run_pair(inst, "f32", 12, **params)


def test_hub_variable_falls_back_to_generic_v2f():
    """max degree > 32: the variable side uses the generic kernel, the factor side stays tiled."""
    inst = random_factor_graph(400, 4, 900, 2, seed=9)
    inst["edge_var"] = inst["edge_var"].copy()
    inst["edge_var"][0:400:2] = 7          # variable 7 becomes a hub of degree ~200
    ev = inst["edge_var"].reshape(-1, 2)
    ev[ev[:, 0] == ev[:, 1], 1] = 8        # keep scopes distinct
    _run_pair(inst, "f32", 6)


def test_generic_and_tiled_paths_agree(monkeypatch):
    from pydcop_b200 import MaxSumEngine, build_layout
    inst = _mixed_instance(1000, 10, 2000, 2, n_unary=200, seed=3)
    L = build_layout(**inst)
    fast = MaxSumEngine(L, precision="f32").init().step(10)
    monkeypatch.setenv("PYDCOP_B200_NO_FAST", "1")
    slow = MaxSumEngine(L, precision="f32").init().step(10)
    for a, b in zip(fast.messages(), slow.messages()):
        assert np.array_equal(a, b)
    assert np.array_equal(fast.values()[0], slow.values()[0])
    assert fast.launch_count > 0 and slow.launch_count > 0


@pytest.mark.parametrize("precision", ["f32", "f64"])
def test_division_free_approx_match_is_exact(precision):
    import ctypes as C
    import torch
    from pydcop_b200 import _cabi
    lib = _cabi.load()
    npdt, tdt = (np.float32, torch.float32) if precision == "f32" else (np.float64, torch.float64)
    rng = np.random.default_rng(0)
    n = 1 << 20
    stab = 0.1
    prev = rng.uniform(-50, 50, n).astype(npdt)
    # c such that 2|prev-c|/|prev+c| lands within a few ulps of stab: c = prev*(2-s)/(2+s) (1+k eps)
    ratio = npdt((2 - stab) / (2 + stab))
    eps = np.finfo(npdt).eps
    k = rng.integers(-6, 7, n)
    c = (prev * ratio * (1 + k * eps)).astype(npdt)
    # sprinkle exact equality, zeros, sign flips, infinities, tiny values
    c[::17] = prev[::17]
    c[1::97] = -prev[1::97]
    prev[2::101] = 0
    c[3::103] = np.inf
    prev[5::107] *= npdt(1e-38 if precision == "f32" else 1e-300)
    c[5::107] *= npdt(1e-38 if precision == "f32" else 1e-300)
    # non-finite operands, as hard constraints produce them: NaN on either side, an infinite previous
    # message, equal infinities, opposite infinities
    prev[7::109] = np.nan
    c[11::113] = np.nan
    prev[13::127], prev[17::131] = np.inf, -np.inf
    prev[19::137], c[19::137] = np.inf, np.inf
    prev[23::139], c[23::139] = -np.inf, -np.inf
    prev[29::149], c[29::149] = np.inf, -np.inf
    prev[31::151], c[31::151] = -np.inf, np.inf
    prev[37::157], c[37::157] = np.nan, np.nan
    dc, dp = torch.from_numpy(c).cuda(), torch.from_numpy(prev).cuda()
    of, oe = torch.zeros(n, dtype=torch.uint8, device="cuda"), torch.zeros(n, dtype=torch.uint8, device="cuda")
    rc = lib.fg_selftest_approx_match(_cabi.FG_F32 if precision == "f32" else _cabi.FG_F64, n,
                                      C.c_void_p(dc.data_ptr()), C.c_void_p(dp.data_ptr()), stab,
                                      C.c_void_p(of.data_ptr()), C.c_void_p(oe.data_ptr()),
                                      C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    torch.cuda.synchronize()
    assert torch.equal(of, oe)
    fin = np.isfinite(prev) & np.isfinite(c)
    match = oe.cpu().numpy().astype(bool)
    frac = float(match[fin].mean())
    assert 0.2 < frac < 0.8, frac   # the finite inputs really straddle the threshold
    # a non-finite pair matches only when both are the same infinity (maxsum.py:688-710: NaN comparisons fail)
    assert np.array_equal(match[~fin], (prev == c)[~fin])


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("variant,mode,d", [("B", "min", 20), ("A", "min", 10), ("C", "max", 5), ("B", "max", 8)])
def test_dsa_binary_fast_path_vs_oracle(variant, mode, d, precision):
    """oriented-table DSA kernel (all constraints binary, one domain size) against the oracle;
    few distinct integer costs -> many ties -> the delta == 0 branches are exercised."""
    from pydcop_b200 import DsaEngine, build_layout
    rng = np.random.default_rng(7)
    inst = random_factor_graph(2500, d, 7000, 2, seed=11 + d, noise=0.0)
    inst["tables"] = rng.integers(0, 3, len(inst["tables"])).astype(np.float32)
    L = build_layout(**inst)
    npdt = np.float64 if precision == "f64" else np.float32
    o = orc.DsaOracle(oracle_instance(inst, L), npdt, mode=mode, variant=variant, seed=31).init()
    eng = DsaEngine(L, precision=precision, mode=mode, variant=variant, seed=31).init()
    assert eng.tables_or is not None          # the fast path is really the one running
    assert np.array_equal(eng.values(), o.val)
    for k in range(12):
        o.step()
        eng.step()
        assert np.array_equal(eng.values(), o.val), k
    assert eng.launch_count > 0
