import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def oracle():
    import oracle_lib
    return oracle_lib.load()


@pytest.fixture(scope="session")
def ref_session():
    import ref_golden
    s = ref_golden.Session()
    yield s
    s.close()


@pytest.fixture
def ref(request, ref_session):
    """The reference's own compiled kernels (oracle/_ref/libjvector.so) where they were built, else a replay of their recorded
    answers to this test's calls (tests/ref_golden.py)."""
    module = os.path.basename(str(request.node.fspath))
    r = ref_session.for_test(module, request.node.name)
    if r is None:
        pytest.fail("no reference library and no recording of its answers for %s::%s" % (module, request.node.name))
    return r


@pytest.fixture(scope="session")
def sift():
    import oracle_lib
    return oracle_lib.load_siftsmall()
