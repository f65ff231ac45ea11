"""Import shims that let the UNMODIFIED reference (pyDcop) import under Python 3.12 / numpy 2.
TEST INFRASTRUCTURE ONLY.

Only the fixture generators (`oracle/make_golden*.py`), the plugin tests, the drop-in test and bench.py's
`reference-threadmode` baseline use this; nothing in the product path imports it.  The reference is
its source tree (PYDCOP_REFERENCE, default /root/reference) where one exists, else the unmodified copy
that `install_copy()` made of it under oracle/_ref (git-ignored build product, made by
__graft_entry__.build()).

Shims (SURVEY.md §8c):
  1. collections.Iterable/Mapping/... aliases (reference: pydcop/dcop/yamldcop.py:32, dcop.py:238)
  2. stub `websocket_server` package (reference: pydcop/infrastructure/ui.py:36)
  3. stub `pulp` package (reference: ILP distributions, commands/generators/iot.py:47-49)
"""
import collections
import collections.abc
import os
import sys
import types

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
#: a pyDcop source tree, when there is one
SOURCE_ROOT = os.environ.get("PYDCOP_REFERENCE") or "/root/reference"
#: the unmodified copy `install_copy()` makes of SOURCE_ROOT (git-ignored)
INSTALLED_ROOT = os.path.join(_REPO, "oracle", "_ref")
#: the reference's test instances (its tests/instances/*.y*ml), stored with this project's fixtures
INSTANCES = os.path.join(_REPO, "tests", "golden", "instances")
REFERENCE_ROOT = SOURCE_ROOT if os.path.isdir(os.path.join(SOURCE_ROOT, "pydcop")) else INSTALLED_ROOT
#: all of the reference's own test instances, with the python files some of them load (only where the reference is)
REFERENCE_INSTANCES = os.path.join(REFERENCE_ROOT, "tests", "instances")


def reference_available() -> bool:
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "pydcop"))


def install() -> None:
    if not reference_available():
        raise RuntimeError(f"reference tree not found at {REFERENCE_ROOT}")
    for n in ("Iterable", "Mapping", "Callable", "Sized", "MutableMapping", "Sequence",
              "Hashable", "Container", "Set", "MutableSet", "MutableSequence"):
        if not hasattr(collections, n):
            setattr(collections, n, getattr(collections.abc, n))
    if "websocket_server" not in sys.modules:
        ws = types.ModuleType("websocket_server")
        ws2 = types.ModuleType("websocket_server.websocket_server")
        ws2.WebsocketServer = type(
            "WebsocketServer", (), {"__init__": lambda self, *a, **k: None})
        ws.websocket_server = ws2
        sys.modules["websocket_server"] = ws
        sys.modules["websocket_server.websocket_server"] = ws2
    if "pulp" not in sys.modules:
        class _Stub(types.ModuleType):
            def __getattr__(self, n):
                if n.startswith("__"):
                    raise AttributeError(n)
                return object
        for name in ("pulp", "pulp.constants", "pulp.pulp", "pulp.solvers"):
            sys.modules[name] = _Stub(name)
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)


def install_copy() -> None:
    """`pip install --no-index --no-deps --target oracle/_ref` of the source tree at SOURCE_ROOT, built from a
    copy under a temporary directory (the source tree may be read-only), plus its tests/instances directory (the
    package does not install it).  Nothing happens without a source tree or when the copy exists; a failed install
    is reported and leaves no copy."""
    import shutil
    import subprocess
    import tempfile
    if not os.path.isdir(os.path.join(SOURCE_ROOT, "pydcop")):
        return
    inst = os.path.join(INSTALLED_ROOT, "tests", "instances")
    if os.path.isdir(os.path.join(INSTALLED_ROOT, "pydcop")) and os.path.isdir(inst):
        return
    with tempfile.TemporaryDirectory() as td:
        cp = os.path.join(td, "ref")
        shutil.copytree(SOURCE_ROOT, cp, ignore=shutil.ignore_patterns(".git", "__pycache__", "docs"))
        for root, dirs, files in os.walk(cp):
            for n in dirs + files:
                os.chmod(os.path.join(root, n), 0o755 if n in dirs else 0o644)
        r = subprocess.run([sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps",
                            "--no-cache-dir", "--target", INSTALLED_ROOT, cp], capture_output=True, text=True)
    if r.returncode != 0:
        shutil.rmtree(INSTALLED_ROOT, ignore_errors=True)
        print("reference install failed (oracle/_ref): " + r.stderr[-400:], file=sys.stderr)
        return
    shutil.copytree(os.path.join(SOURCE_ROOT, "tests", "instances"), inst, dirs_exist_ok=True)
