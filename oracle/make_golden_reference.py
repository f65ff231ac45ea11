"""What the UNMODIFIED reference says about its own test instances and algorithm parameters.

TEST INFRASTRUCTURE ONLY.  Needs the reference (oracle/ref_shim.py):

    python oracle/make_golden_reference.py

For every instance under tests/golden/instances/ (the reference's tests/instances/*.y*ml) it records what
the reference's `load_dcop_from_file` makes of it: the variable and constraint names in the reference's
order, whether it has external variables, whether a variable carries noise, and every constraint's table
with its axes in sorted variable-name order (make_golden_ingest.describe).  It also records the names,
defaults and allowed values of the `algo_params` of the reference's maxsum, dsa and mgm modules.
Output: tests/golden/reference_expected.json (names, scopes, parameters) and reference_tables.npz (the
tables, float64, keyed "<instance file>/<constraint name>"), read by tests/test_ingest.py and
tests/test_solve_cpu.py.
"""
import glob
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)


def main():
    import ref_shim
    ref_shim.install()
    from pydcop.algorithms import load_algorithm_module
    from pydcop.dcop.yamldcop import load_dcop_from_file
    from make_golden_ingest import describe
    instances, tables = {}, {}
    for fn in sorted(glob.glob(os.path.join(ref_shim.INSTANCES, "*.y*ml"))):
        ref = load_dcop_from_file([fn])  # a bare str is iterated char by char (yamldcop.py:85)
        entry = {"external_variables": bool(ref.external_variables)}
        if not ref.external_variables:
            entry.update(var_names=list(ref.variables), con_names=list(ref.constraints),
                         noise=any(hasattr(v, "noise_level") for v in ref.variables.values()),
                         scopes={})
            for cn, c in describe(ref)["constraints"].items():
                entry["scopes"][cn] = c["scope"]
                tables[os.path.basename(fn) + "/" + cn] = np.asarray(c["table"], np.float64)
        instances[os.path.basename(fn)] = entry
    algo_params = {}
    for name in ("maxsum", "dsa", "mgm"):
        algo_params[name] = {p.name: {"default": p.default_value, "values": list(p.values) if p.values else None}
                             for p in load_algorithm_module(name).algo_params}
    path = os.path.join(ROOT, "tests", "golden", "reference_expected.json")
    with open(path, "w") as f:
        json.dump({"instances": instances, "algo_params": algo_params}, f, indent=1, sort_keys=True)
        f.write("\n")
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "reference_tables.npz"), **tables)
    print("wrote", path, len(instances), "instances,", len(tables), "tables")


if __name__ == "__main__":
    main()
