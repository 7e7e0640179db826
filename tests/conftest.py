import os, sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); run with -m gpu on a machine that has one")


@pytest.fixture(scope="session")
def oracle():
    from tests.orc import Oracle, IMAGE
    if not os.path.exists(IMAGE):
        pytest.skip("model image missing: run __graft_entry__.build() where /root/reference exists")
    o = Oracle(IMAGE)
    yield o
    o.close()


@pytest.fixture(scope="session")
def oracle_cong():
    from tests.orc import Oracle, CONG_IMAGE
    if not os.path.exists(CONG_IMAGE):
        pytest.skip("CoNg model image missing: run __graft_entry__.build() where /root/reference exists")
    o = Oracle(CONG_IMAGE)
    yield o
    o.close()


@pytest.fixture(scope="session")
def oracle_sbg():
    from tests.orc import Oracle, SBG_IMAGE
    if not os.path.exists(SBG_IMAGE):
        pytest.skip("SkipBigram model image missing: run __graft_entry__.build() where /root/reference exists")
    o = Oracle(SBG_IMAGE)
    yield o
    o.close()


@pytest.fixture(scope="session")
def kiwi_cong():
    import kiwi_b200
    from tests.orc import CONG_IMAGE
    kw = kiwi_b200.Kiwi(CONG_IMAGE)
    yield kw
    kw.close()


@pytest.fixture(scope="session")
def kiwi():
    import kiwi_b200
    from tests.orc import IMAGE
    kw = kiwi_b200.Kiwi(IMAGE)      # raises when the CUDA extension or the GPU is missing: no fallback
    yield kw
    kw.close()
