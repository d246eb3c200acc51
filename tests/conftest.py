import os
import sys

import pytest

os.environ.setdefault("OMP_NUM_THREADS", "4")   # the oracle's XNNPACK shim uses OpenMP; keep it from fanning out over every core

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

ORACLE_LIB = os.path.join(ROOT, "oracle", "_ref", "liboracle_ref.so")
ENGINE_LIB = os.path.join(ROOT, "onnxstream_b200", "csrc", "libonnxstream_b200.so")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with `-m gpu`)")


@pytest.fixture(scope="session")
def oracle_lib():
    """The reference built in place (oracle/Makefile), or None: the parity tests then compare with the stored reference
    outputs under tests/golden/oracle (tests/util.py)."""
    return ORACLE_LIB if os.path.exists(ORACLE_LIB) else None


@pytest.fixture(scope="session")
def engine_lib():
    assert os.path.exists(ENGINE_LIB), "libonnxstream_b200.so not built: run __graft_entry__.build()"
    return ENGINE_LIB
