import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu)")


def _ensure_built():
    import __graft_entry__ as ge
    ge.build()


@pytest.fixture(scope="session")
def zq():
    _ensure_built()
    import zpaqfranz_b200
    return zpaqfranz_b200


@pytest.fixture(scope="session")
def ctx(zq):
    c = zq.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="session")
def oracle():
    """oracle/_ref/libzqoracle.so -- this repo's plain-C restatement (the checker)."""
    _ensure_built()
    import oracle_bindings
    return oracle_bindings.load_oracle()


@pytest.fixture(scope="session")
def ref(oracle):
    """The reference's answers (zpaqfranz's own libzpaq): replayed from tests/golden/ref_answers.json.  With
    ZQ_REF_RECORD=<path> they come from the live reference in oracle/_ref/libzpaqref.so and are written to <path>."""
    import oracle_bindings
    path = os.environ.get("ZQ_REF_RECORD")
    if not path:
        yield oracle_bindings.load_recorded_ref(oracle)
        return
    live = oracle_bindings.load_ref()
    if live is None:
        pytest.fail("ZQ_REF_RECORD is set but oracle/_ref/libzpaqref.so is not built")
    r = oracle_bindings.RecordingRef(live)
    yield r
    r.save(path)
