import os
import sys

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_sessionstart(session):
    """Built artefacts are git-ignored: (re)build the C-ABI library, the host packer and the CPU oracle when they are
    missing or older than their sources (a no-op when build() already made them)."""
    from polyfuzz_b200 import build as b
    from oracle import native
    native.build()                                          # gcc only
    b.build_hostpack()                                      # gcc only
    try:
        b.build(force=False)                                # nvcc (cross-compiles sm_90a without a GPU)
    except (RuntimeError, OSError) as e:
        import torch
        if torch.cuda.is_available() or "gpu" in (session.config.getoption("-m") or ""):
            raise                                           # a GPU run must never continue without the CUDA library
        session.config._pfz_build_error = str(e)            # CPU-only box without nvcc: oracle / host-logic tests still run


def pytest_collection_modifyitems(config, items):
    """GPU tests must never silently pass on a box without a GPU: they are skipped only when CUDA is
    absent AND -m gpu was not requested; with -m gpu on a GPU-less box they fail loudly."""
    import torch
    if torch.cuda.is_available():
        return
    requested = "gpu" in (config.getoption("-m") or "")
    if requested:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
