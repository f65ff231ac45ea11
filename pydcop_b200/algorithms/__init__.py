"""pyDcop algorithm modules backed by the GPU engine.

This directory is appended to `pydcop.algorithms.__path__` (see pydcop_b200.launcher.install),
after which the unmodified reference lists and loads `maxsum_gpu` / `dsa_gpu` like its own
algorithms (pydcop/algorithms/__init__.py:508-566)."""
