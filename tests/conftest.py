import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def port():
    import oracle_lib as O
    return O.Port()


@pytest.fixture(scope="session")
def ref():
    import oracle_lib as O
    if not O.have_ref():
        O.build_ref()
    if not O.have_ref():
        pytest.skip("oracle/_ref not built and the reference source tree is not readable")
    return O.Ref()


@pytest.fixture(scope="session")
def pkg():
    import pkgload
    return pkgload.load()


@pytest.fixture(scope="session")
def lib(pkg):
    return pkg.Lib.get()


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch.device("cuda:0")
