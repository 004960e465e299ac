"""pytest configuration: the `gpu` marker and shared fixtures.

`-m "not gpu"`: oracle vs golden vectors / vs the compiled reference, host logic, C-ABI symbol
checks.  `-m gpu`: parity tests proper, through the C-ABI on a real H100.
"""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


def pytest_collection_modifyitems(config, items):
    """A plain `pytest tests` on a box without a CUDA device skips the gpu-marked tests instead of failing in them (the
    product has no CPU path to fall back to: every entry point returns PGEMB_ERR_CUDA there)."""
    if not any("gpu" in it.keywords for it in items):
        return
    try:
        from pg_embedding_b200 import _lib
        have = _lib.load().pgemb_device_count() > 0
    except Exception:
        return          # a missing / unloadable extension must FAIL the gpu tests loudly, never skip them
    if have:
        return
    skip = pytest.mark.skip(reason="no CUDA device (pgemb_device_count() == 0); run with -m gpu on an H100")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def oracle_mod():
    from oracle import oracle

    oracle.build("all")
    return oracle


@pytest.fixture(scope="session")
def have_ref(oracle_mod):
    return oracle_mod.available("ref")


def checker_names(oracle_mod):
    names = ["port"]
    if oracle_mod.available("ref"):
        names.append("ref")
    return names
