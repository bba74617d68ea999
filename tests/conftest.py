import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a machine that has one)")


def pytest_collection_modifyitems(config, items):
    # `-m gpu` on a box without CUDA is a usage error, not a silent pass
    pass


def _has_cuda() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


HAS_CUDA = _has_cuda()


@pytest.fixture(scope="session")
def oracle_mod():
    import oracle
    oracle.build()
    return oracle


@pytest.fixture(scope="session")
def native():
    # building is idempotent; on the GPU box the prebuilt .so is used as is
    import importlib.util
    spec = importlib.util.spec_from_file_location("rbk_build", ROOT / "runbookai_b200" / "build.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    if mod.needs_build() and os.environ.get("RBK_NO_REBUILD") != "1":
        mod.build()
    from runbookai_b200 import _native
    return _native
