"""The unions of tests/test_gpu_zz_binary_paths.py without a GPU: every one takes the binary kernels at its domain size,
its blocks of 128 variables mix problems (and parameter sets), its hub has more slots than an active-row chunk, its
keys and sets are the ones intended, and its oracle trajectories show what the GPU test relies on: the copies
diverge, the probability-0 problem stays put, and variables move early and late."""
import os
import re

import numpy as np
import pytest
import torch

import _binary_unions as bu
from pydcop_b200 import batch
from pydcop_b200.engine import dsa_fast_arrays
from pydcop_b200.solve import check_params

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ([("dsa", D, m) for D in bu.FAST_DOMS for m in (True, False)] + [("adsa", D, True) for D in (2, 5, 10, 20)]
         + [("mgm", D, False) for D in bu.MGM_DOMS])


def test_domain_sizes_are_the_compiled_ones():
    with open(os.path.join(ROOT, "pydcop_b200", "csrc", "maxsum_fast.cuh")) as f:
        doms = re.search(r"#define FG_FAST_DOMS\(X\)(.*)", f.read()).group(1)
    assert tuple(int(x) for x in re.findall(r"X\((\d+)\)", doms)) == bu.FAST_DOMS


def _union(kind, D, mixed):
    dcops, params, seeds = bu.case(kind, D, mixed)
    checked = None if params is None else [check_params(kind, p) for p in params]
    u = batch.build_union(dcops, list(range(len(dcops))), lambda d: (None, None), seed=seeds, params=checked)
    return dcops, u, batch.union_layout(u, dcops)


@pytest.mark.parametrize("kind,D,mixed", CASES)
def test_union_takes_the_binary_kernels(kind, D, mixed):
    dcops, u, L = _union(kind, D, mixed)
    fast = dsa_fast_arrays(L, torch.from_numpy(np.ascontiguousarray(L.tables, np.float32)), dcops[0].objective)
    assert fast is not None and fast[4] == D        # one class: binary over domain size D
    assert len(dcops) == 7 and all(d.objective == dcops[0].objective for d in dcops)
    assert not (np.diff(u.var_start) % bu.CTA == 0).any()
    deg = np.diff(L.canon_var_ptr)
    hub = kind == "mgm" or D in bu.HUB_DOMS
    a, b = u.var_start[bu.HUB], u.var_start[bu.HUB + 1]
    assert (deg[a:b].max() >= bu.HUB_DEGREE) == hub and (deg.max() >= bu.HUB_DEGREE) == hub
    assert bu.HUB_DEGREE > 128 * 8                  # the largest active-row chunk: 128 threads x 8 slots
    assert ((deg == 0) & (u.seg_var == 0)).sum() >= bu.ISOLATED[0]
    # kernel blocks run over the internal order: some hold variables of several problems, with different sets
    blocks = np.arange(L.n_vars) // bu.CTA
    seg = u.seg_var[L.var_order]
    mixed_blocks = np.unique(blocks[np.r_[False, (seg[1:] != seg[:-1]) & (blocks[1:] == blocks[:-1])]])
    assert len(mixed_blocks) >= 2
    keys = np.unique(u.var_seed)
    assert len(keys) >= 2 and {0, 2 ** 63, 2 ** 64 - 1} <= {int(k) for k in keys}
    if mixed:
        assert len(np.unique(u.var_pset)) == len(u.psets) == 7
        ps = u.var_pset[L.var_order]
        assert any(len(np.unique(ps[blocks == k])) > 1 for k in mixed_blocks)
    else:
        assert u.var_pset is None


@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("kind,D,mixed", CASES)
def test_oracle_trajectories_are_not_vacuous(kind, D, mixed, precision):
    bu.check_non_vacuous(kind, bu.case_trajectories(kind, D, mixed, precision, 30), mixed)


def test_copies_are_one_instance_with_one_start():
    dcops, _, _ = bu.case("mgm", 10, False)
    a, b, c = (dcops[i] for i in bu.COPIES)
    assert a is b is c and (a.arrays["init_value"] >= 0).all()
    _, params, seeds = bu.case("dsa", 10, True)
    assert len({seeds[i] for i in bu.COPIES}) == 1 and [params[i]["variant"] for i in bu.COPIES] == ["A", "C", "B"]
    assert len({params[i]["probability"] for i in bu.COPIES}) == 1 and params[bu.FROZEN]["probability"] == 0.0
    others = [s for i, s in enumerate(seeds) if i not in bu.COPIES]
    assert len(set(others + [seeds[bu.COPIES[0]]])) == len(others) + 1
