import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def port():
    """The C oracle port (oracle/msm_oracle.c), built on demand with gcc."""
    from oracle import port as p
    p.build()
    return p


@pytest.fixture(scope="session")
def _reference_store():
    from tests import recorded_reference as rr
    store = rr.Store()
    yield store
    if os.environ.get("BLITZAR_RECORD_REFERENCE"):
        store.save(os.environ["BLITZAR_RECORD_REFERENCE"])


def _reference(store, label, module):
    from tests import recorded_reference as rr
    return rr.RecordedReference(label, module if module.available() else None, store)


@pytest.fixture(scope="session")
def refcpu(_reference_store):
    """The reference's own CPU path (oracle/_ref) when built, else its recorded answers."""
    from oracle import refcpu as r
    return _reference(_reference_store, "refcpu", r)


@pytest.fixture(scope="session")
def refgpu(_reference_store):
    """The reference's own GPU bucket kernels (oracle/_ref) when built, else their recorded answers."""
    from oracle import refgpu as r
    return _reference(_reference_store, "refgpu", r)


@pytest.fixture(scope="session")
def emul():
    """CPU emulation of the product's kernel bodies (tests/emul) — test infrastructure."""
    from tests.emul import harness
    return harness


@pytest.fixture(scope="session")
def bb():
    """The product library, initialised on the GPU."""
    import blitzar_b200 as b
    assert b.sxt_init(num_precomputed_generators=64) == 0
    return b
