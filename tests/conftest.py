import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "d-liom_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); select with -m gpu")
    # a fresh checkout has no built artefacts (*.so are git-ignored): build the product library and the oracle once
    lib = os.path.join(ROOT, "d-liom_b200", "libdliom_b200.so")
    orc_lib = os.path.join(ROOT, "oracle", "build", "liborc.so")
    if not (os.path.exists(lib) and os.path.exists(orc_lib)):
        import __graft_entry__
        __graft_entry__.build()


@pytest.fixture(scope="session")
def orc():
    import orc as _orc
    _orc.lib()
    return _orc
