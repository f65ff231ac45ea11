"""The host shims of tests/hostshim/: each compiles a family's kernel headers with g++ and runs the entry points'
own launch sequences on the CPU, one "thread" after the other (tests/hostshim/cuda_host.h).  build() compiles and
caches a shim; HostRun drives an engine's host-array plan through a descriptor family's shim."""
import ctypes as C
import functools
import os
import subprocess

from conftest import ROOT
from pydcop_b200 import _cabi
from pydcop_b200.engine import _class_array, fill_desc, fill_header, host_state

CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
SHIMS = os.path.join(ROOT, "tests", "hostshim")
BUILD = os.path.join(SHIMS, "_build")


def _deps(src):
    csrc = os.path.join(ROOT, "pydcop_b200", "csrc")
    return [src, os.path.join(SHIMS, "cuda_host.h"), os.path.join(ROOT, "include", "pydcop_b200.h")] + [
        os.path.join(csrc, f) for f in os.listdir(csrc)]


@functools.lru_cache(maxsize=None)
def build(name):
    """tests/hostshim/<name>.cpp as a loaded shared library, rebuilt under tests/hostshim/_build/ when the shim,
    cuda_host.h, a file of pydcop_b200/csrc/ or include/pydcop_b200.h is newer.  Every <family>_host_* entry point
    returns the launches it ran (int64)."""
    src = os.path.join(SHIMS, name + ".cpp")
    so = os.path.join(BUILD, name + ".so")
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in _deps(src)):
        os.makedirs(BUILD, exist_ok=True)
        gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        tmp = f"{so}.{os.getpid()}"   # several test processes may build at once
        subprocess.run([gxx, "-O1", "-std=c++17", "-ffp-contract=off", "-I", CUDA_INC, "-shared", "-fPIC", "-o", tmp,
                        src], check=True, capture_output=True)
        os.replace(tmp, so)
    lib = C.CDLL(so)
    for fn in ("init", "cycle", "phase", "unpack"):
        for family in ("dsa", "mgm", "mgm2", "gdba", "mixeddsa", "dba", "mgm2_shard"):
            if hasattr(lib, f"{family}_host_{fn}"):
                getattr(lib, f"{family}_host_{fn}").restype = C.c_int64
    return lib


DESCS = dict(dsa=_cabi.FgDsaDesc, mgm=_cabi.FgMgmDesc, mgm2=_cabi.FgMgm2Desc, gdba=_cabi.FgGdbaDesc,
             mixeddsa=_cabi.FgMixedDsaDesc, dba=_cabi.FgDbaDesc)
SHIM = dict(dsa="dsa_generic_host", mgm="mgm_host", mgm2="mgm2_host", gdba="gdba_host", mixeddsa="mixeddsa_host",
            dba="dba_host")


class HostRun:
    """An engine's host-array plan (inputs, state, scalars) in the family's C-ABI descriptor with host pointers, run
    by the family's shim: init() and step() as the engines', stopping as fg_<family>_step does (DSA and MixedDSA once
    cycle >= stop_cycle, the others once cycle + 1 >= stop_cycle).  `rounds` counts the rounds run, `launches` what
    the shim launched."""

    def __init__(self, family, layout, plan, precision):
        inputs, state, scalars = plan
        self.family, self.L = family, layout
        self.lib = build(SHIM[family])
        self.k = dict(inputs, **host_state(state))
        self.classes = _class_array(layout)
        self.d = fill_desc(fill_header(DESCS[family](), precision, layout, self.classes), self.k, scalars)
        self.stop_cycle, self.rounds, self.launches = int(scalars.get("stop_cycle", 0)), 0, 0

    @property
    def cycle(self):
        return self.rounds

    @property
    def finished(self):
        last = self.rounds if self.family in ("dsa", "mixeddsa") else self.rounds + 1
        return bool(self.stop_cycle and last >= self.stop_cycle)

    def _run(self, fn, *args):
        n = getattr(self.lib, f"{self.family}_host_{fn}")(C.byref(self.d), *args)
        assert n >= 0, f"{self.family}_host_{fn} refused the descriptor"
        self.launches += n

    def init(self):
        self._run("init")
        self.rounds = 0
        return self

    def step(self, n=1):
        for _ in range(n):
            if self.finished:
                break
            self._run("cycle", C.c_int64(self.rounds))
            self.rounds += 1
        return self

    @property
    def value(self):
        """The current values, internal order: the buffer of the double-buffered families' current round."""
        v = self.k["value"]
        return v[self.rounds % 2] if isinstance(v, list) else v
