#!/usr/bin/env python
"""Extra MaxSum trajectories from the UNMODIFIED reference for cases the main fixture set does not
hold: infinite (hard-constraint) costs.  Same lock-step method as oracle/make_golden.py.

TEST INFRASTRUCTURE (build container only).  Fixtures are written with the prefix `msx_`.  The CPU
tests run them through the oracle and through the generic kernel source (host shim);
tests/test_gpu_parity.py runs them through every factor-kernel configuration on the device.

Forbidden assignments are +inf cells (min mode) or -inf cells (max mode).  A unary constraint whose
whole row is infinite forbids every value of its variable: that variable's q rows become
inf - inf = NaN in the normalisation, and every marginal a factor computes from such a row has only
NaN candidates.  The reference keeps its +/-inf start value there (maxsum.py:419-445), so each
fixture is built to reach that corner on one factor-kernel site (tests/_hard_constraints.py lists
the sites; tests/test_hard_constraint_fixtures.py checks that every fixture reaches its own):

    msx_hard_inf_{min,max}    binary / ternary / unary over D in {3, 4}
    msx_warp_d4_{min,max}     binary D = 4 (warp kernel, row pairs); variable degrees 1..8, 9..16 and a hub > 16
    msx_warp_d10              binary D = 10 (warp kernel, row pairs and the odd half row)
    msx_pipe_bin_d2_d5        binary D = 2 and D = 5 (pipelined kernel, arity 2), unary all-inf rows
    msx_pipe_tern_{min,max}   ternary D = 3 and D = 4 (pipelined kernel, arity 3)
    msx_tiled_rt_mixed        domains {2, 3, 5, 7}, arities 1..4, arity 7 and 8 over D = 2, one binary D = 40
    msx_p_*                   binary D = 4 with damping_nodes="none", stability=1e-4, start_messages="all"

Tables are integers, so that most value selections are exact.  The reference sums the received costs in
message arrival order, which is not fixed from run to run; the seeds are chosen so that no selection is a
tie that the rounding of that sum decides.

    python oracle/make_golden_extra.py [name ...]
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as G  # noqa: E402


def hard_instance(rng, sign, doms, scopes, dead, inf_every=2, inf_share=0.3):
    """Variables v000.. with domain sizes `doms`; one integer(0, 10) table per scope, about `inf_share`
    of the cells of every `inf_every`-th table set to sign * inf; a unary constraint with a whole row
    of sign * inf on every variable of `dead`."""
    by_size = {}
    variables = []
    for i, d in enumerate(doms):
        if d not in by_size:
            by_size[d] = G.Domain(f"d{d}", "", list(range(d)))
        variables.append(G.Variable(f"v{i:03d}", by_size[d]))
    constraints = []
    for j, scope in enumerate(scopes):
        sv = [variables[int(i)] for i in scope]
        m = rng.integers(0, 10, size=tuple(len(v.domain) for v in sv)).astype(np.float64)
        if j % inf_every == 0:
            m[rng.random(m.shape) < inf_share] = sign * np.inf
        constraints.append(G.NAryMatrixRelation(sv, m, name=f"c{j:03d}"))
    for k, i in enumerate(dead):
        v = variables[int(i)]
        constraints.append(G.NAryMatrixRelation([v], np.full(len(v.domain), sign * np.inf), name=f"u{k:03d}"))
    return variables, constraints


def scopes_over(rng, pool, arity, n):
    """`n` scopes of `arity` distinct variables drawn from `pool`."""
    return [tuple(int(x) for x in rng.choice(pool, size=arity, replace=False)) for _ in range(n)]


def warp_d4(rng, sign, n_vars=30):
    """Binary D = 4; variable 0 is a hub (degree > 16: generic variable kernel), variables 1 and 2 have
    degree 9..16, the others 1..8."""
    pool = np.arange(n_vars)
    scopes = scopes_over(rng, pool[3:], 2, 40)
    scopes += [(0, int(x)) for x in rng.choice(pool[3:], 20, replace=False)]
    scopes += [(v, int(x)) for v in (1, 2) for x in rng.choice(pool[3:], 9, replace=False)]
    rng.shuffle(scopes)
    return hard_instance(rng, sign, [4] * n_vars, scopes, dead=(3, 7, 12))


def main():
    only = set(sys.argv[1:])

    def want(n):
        return not only or n in only

    for name, mode, sign in (("msx_hard_inf_min", "min", 1.0), ("msx_hard_inf_max", "max", -1.0)):
        if not want(name):
            continue
        rng = np.random.default_rng(50)
        vs, cs = G.random_instance(rng, 14, [3, 4], 18, [2, 2, 3, 1])
        for k, c in enumerate(cs):       # a third of the constraints forbid some assignments
            if k % 3 == 0:
                m = c._m
                mask = rng.random(m.shape) < 0.3
                m[mask] = sign * np.inf
        arr, meta = G.run_maxsum(vs, cs, {"noise": 0.0}, mode, 20, seed=51)
        G.save(name, arr, meta)

    for name, mode, sign in (("msx_warp_d4_min", "min", 1.0), ("msx_warp_d4_max", "max", -1.0)):
        if want(name):
            vs, cs = warp_d4(np.random.default_rng(60), sign)
            arr, meta = G.run_maxsum(vs, cs, {"noise": 0.0}, mode, 22, seed=61)
            G.save(name, arr, meta)

    if want("msx_warp_d10"):
        rng = np.random.default_rng(64)
        vs, cs = hard_instance(rng, 1.0, [10] * 24, scopes_over(rng, np.arange(24), 2, 40), dead=(2, 9, 17))
        arr, meta = G.run_maxsum(vs, cs, {"noise": 0.0}, "min", 20, seed=65)
        G.save("msx_warp_d10", arr, meta)

    if want("msx_pipe_bin_d2_d5"):
        rng = np.random.default_rng(64)
        doms = [2] * 16 + [5] * 16
        scopes = scopes_over(rng, np.arange(16), 2, 26) + scopes_over(rng, np.arange(16, 32), 2, 26)
        vs, cs = hard_instance(rng, 1.0, doms, scopes, dead=(1, 6, 18, 25))
        arr, meta = G.run_maxsum(vs, cs, {"noise": 0.0}, "min", 20, seed=65)
        G.save("msx_pipe_bin_d2_d5", arr, meta)

    for name, mode, sign in (("msx_pipe_tern_min", "min", 1.0), ("msx_pipe_tern_max", "max", -1.0)):
        if want(name):
            rng = np.random.default_rng(66)
            doms = [3] * 14 + [4] * 14
            scopes = scopes_over(rng, np.arange(14), 3, 14) + scopes_over(rng, np.arange(14, 28), 3, 14)
            vs, cs = hard_instance(rng, sign, doms, scopes, dead=(2, 9, 16, 23))
            arr, meta = G.run_maxsum(vs, cs, {"noise": 0.0}, mode, 20, seed=67)
            G.save(name, arr, meta)

    if want("msx_tiled_rt_mixed"):
        rng = np.random.default_rng(68)
        # 0..23: domains {2, 3, 5, 7}; 24..33: D = 2 (arity 7 and 8); 34, 35: D = 40 (one binary factor wider than a warp)
        doms = [int(x) for x in rng.choice([2, 3, 5, 7], size=24)] + [2] * 10 + [40, 40]
        mixed = np.arange(24)
        scopes = []
        for a, n in ((1, 3), (2, 14), (3, 8), (4, 4)):
            scopes += scopes_over(rng, mixed, a, n)
        scopes += scopes_over(rng, np.arange(20, 34), 7, 2) + scopes_over(rng, np.arange(20, 34), 8, 2)
        scopes += [(34, 35), (34, int(rng.choice(mixed)))]
        vs, cs = hard_instance(rng, 1.0, doms, scopes, dead=(4, 11, 26, 29, 35))
        arr, meta = G.run_maxsum(vs, cs, {"noise": 0.0}, "min", 20, seed=69)
        G.save("msx_tiled_rt_mixed", arr, meta)

    sweeps = {
        "msx_p_nodamp": {"damping_nodes": "none"},
        "msx_p_stab_tiny": {"stability": 1e-4},
        "msx_p_start_all": {"start_messages": "all"},
    }
    for name, params in sweeps.items():
        if want(name):
            vs, cs = warp_d4(np.random.default_rng(70), 1.0, n_vars=24)
            arr, meta = G.run_maxsum(vs, cs, dict(params, noise=0.0), "min", 20, seed=71)
            G.save(name, arr, meta)


if __name__ == "__main__":
    main()
