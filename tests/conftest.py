import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); select with -m gpu")


def load_golden(name: str) -> dict:
    with open(os.path.join(GOLDEN, name)) as f:
        return json.load(f)


@pytest.fixture(scope="session")
def golden():
    return load_golden


@pytest.fixture
def fake_backend(monkeypatch):
    """Host-logic tests on CPU: route the host layer to the oracle-backed stand-in (tests/fake_backend.py)."""
    from modal_client_b200 import _backend
    from tests.fake_backend import FakeContext

    ctx = FakeContext()
    monkeypatch.setattr(_backend, "_override", ctx)
    return ctx


@pytest.fixture
def gpu_backend(monkeypatch):
    """GPU tests: the host layer talks to the real library on cuda:0."""
    from modal_client_b200 import _backend, _lib

    ctx = _lib.Context(0, pinned_bytes=64 << 20, device_bytes=512 << 20)
    monkeypatch.setattr(_backend, "_override", ctx)
    yield ctx
    ctx.close()
