"""CPU: the rule that decides which table entries the factor kernel may store as 8-bit codes
(pydcop_b200/csrc/table_i8.cuh, fg_table_entry_fits_i8), compiled with g++ from the kernel header itself.
An entry qualifies when its signed byte decodes back to the same bits: an integer in [-128, 127], not -0.0."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "pydcop_b200", "csrc", "table_i8.cuh")

SRC = r"""
#include <stdio.h>
#include <stdlib.h>
#define __host__
#define __device__
#include "%s"
int main(int argc, char **argv) {
  // each argument: a hexadecimal bit pattern of a double; prints the rule for it as a double and as a float
  for (int i = 1; i < argc; ++i) {
    unsigned long long b = strtoull(argv[i], 0, 16);
    double x;
    __builtin_memcpy(&x, &b, 8);
    printf("%%d %%d\n", (int)fg_table_entry_fits_i8<double>(x), (int)fg_table_entry_fits_i8<float>((float)x));
  }
  return 0;
}
"""

CASES = [
    (0.0, True), (-0.0, False), (1.0, True), (-1.0, True), (9.0, True), (-128.0, True), (127.0, True),
    (128.0, False), (-129.0, False), (-128.5, False), (127.5, False), (0.5, False), (-0.5, False),
    (1e-45, False), (-1e-45, False), (5e-324, False), (np.finfo(np.float64).tiny, False),
    (float("nan"), False), (-float("nan"), False), (float("inf"), False), (-float("inf"), False),
    (2.0 ** 31, False), (-(2.0 ** 31) - 1, False), (1e300, False), (127.00000000000001, False),
]


@pytest.fixture(scope="module")
def rule_exe(tmp_path_factory):
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not available")
    d = tmp_path_factory.mktemp("table_i8")
    src, exe = d / "rule.cpp", d / "rule"
    src.write_text(SRC % HEADER)
    subprocess.run([gxx, "-O2", "-std=c++17", "-o", str(exe), str(src)], check=True, capture_output=True)
    return str(exe)


def test_rule_edge_cases(rule_exe):
    bits = [format(np.array(x, dtype=np.float64).view(np.uint64).item(), "x") for x, _ in CASES]
    out = subprocess.run([rule_exe, *bits], check=True, capture_output=True, text=True).stdout.split("\n")
    for (x, want), line in zip(CASES, out):
        as_double, as_float = (bool(int(t)) for t in line.split())
        assert as_double == want, (x, "f64")
        with np.errstate(over="ignore"):
            xf = np.float32(x)   # 1e300 becomes inf, as the C cast does
        want_f = bool(np.isfinite(xf) and xf == np.rint(xf) and -128 <= xf <= 127 and not (xf == 0 and np.signbit(xf)))
        assert as_float == want_f, (x, "f32")


def test_rule_matches_int8_round_trip(rule_exe):
    """Over every integer in [-200, 200] and values near them: qualifies exactly when the byte round trip keeps
    the bits."""
    xs = np.concatenate([np.arange(-200, 201, dtype=np.float64), np.arange(-200, 201) + 0.25,
                         np.nextafter(np.arange(-130, 131, dtype=np.float64), np.inf)])
    bits = [format(np.array(x).view(np.uint64).item(), "x") for x in xs]
    out = subprocess.run([rule_exe, *bits], check=True, capture_output=True, text=True).stdout.split("\n")
    for x, line in zip(xs, out):
        got = bool(int(line.split()[0]))
        rt = -128 <= x <= 127 and float(np.int8(x) if -128 <= x <= 127 else 0) == x
        want = bool(rt) and np.array(float(np.int8(x)) if rt else 0.0).view(np.uint64) == np.array(x).view(np.uint64)
        assert got == bool(want), x
