"""pytest configuration: the `gpu` marker and import paths.

* `-m "not gpu"` (runs on the CPU-only build box): oracle vs the golden vectors, host logic, the C-ABI
  library loads and exports every declared symbol, gloo world_size-2 sharding tests.
* `-m gpu` (runs on an H100): the parity tests proper, through the C ABI / Python drop-in API.
"""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "wild-gaussians_b200"), os.path.join(ROOT, "tests", "golden")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    # Make sure the in-tree libraries are up to date BEFORE any test module imports (and dlopens) them
    # (no-op when they are newer than their sources).
    import __graft_entry__ as ge
    ge.build_lib()
    from oracle import cpu_oracle
    cpu_oracle.build()


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
