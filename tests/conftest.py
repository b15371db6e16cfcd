import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "fast-lio-sam-qn_b200"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA GPU (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as orc
    orc.lib()
    return orc


@pytest.fixture(scope="session")
def synth():
    from b200reg import synth as s
    return s


@pytest.fixture(scope="session")
def native():
    from b200reg import native as n
    return n


@pytest.fixture(scope="session")
def ctx():
    import b200reg
    c = b200reg.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="session")
def pair20k(synth):
    return synth.make_pair(1000, 20000)


@pytest.fixture(scope="session")
def pair5k(synth):
    return synth.make_pair(1001, 5000, 6000)
