import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")


def _import_pkg():
    """The package directory is named caesium-clt_b200 (not an identifier); import it under caesium_clt_b200."""
    import importlib.util
    if "caesium_clt_b200" in sys.modules:
        return sys.modules["caesium_clt_b200"]
    pkg_dir = os.path.join(ROOT, "caesium-clt_b200")
    spec = importlib.util.spec_from_file_location("caesium_clt_b200", os.path.join(pkg_dir, "__init__.py"), submodule_search_locations=[pkg_dir])
    mod = importlib.util.module_from_spec(spec)
    sys.modules["caesium_clt_b200"] = mod
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="session")
def L():
    _import_pkg()
    import caesium_clt_b200._lib as lib
    if not os.path.exists(lib.LIB_PATH):
        lib.build()
    lib.lib()
    return lib


@pytest.fixture(scope="session")
def O():
    from oracle import oracle
    oracle.lib()
    return oracle


@pytest.fixture(scope="session")
def golden():
    def load(name):
        with open(os.path.join(GOLDEN, name), "rb") as f:
            return f.read()
    return load
