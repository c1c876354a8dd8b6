import importlib.util
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


def load_pkg():
    """Import the hyphenated package directory `karpenter-core_b200` as module `karpenter_core_b200`."""
    if "karpenter_core_b200" in sys.modules:
        return sys.modules["karpenter_core_b200"]
    spec = importlib.util.spec_from_file_location(
        "karpenter_core_b200", ROOT / "karpenter-core_b200" / "__init__.py",
        submodule_search_locations=[str(ROOT / "karpenter-core_b200")])
    mod = importlib.util.module_from_spec(spec)
    sys.modules["karpenter_core_b200"] = mod
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="session")
def pkg():
    return load_pkg()


@pytest.fixture(scope="session")
def oracle():
    import oracle_lib
    return oracle_lib.load()
