import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
if os.path.dirname(os.path.abspath(__file__)) not in sys.path:
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (an H100)")


@pytest.fixture(scope="session", autouse=True)
def _built_library():
    # The native library must exist before anything imports heyoka_b200 (nvcc cross-compiles without a GPU).
    lib = os.path.join(ROOT, "heyoka_b200", "lib", "libheyoka_b200.so")
    if not os.path.exists(lib):
        sys.path.insert(0, os.path.join(ROOT, "heyoka_b200"))
        import importlib.util
        spec = importlib.util.spec_from_file_location("hb_build", os.path.join(ROOT, "heyoka_b200", "build.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod.build(verbose=False)
    yield


@pytest.hookimpl(hookwrapper=True)
def pytest_runtest_call(item):
    # Tests parametrised over kernel shapes force a kernel with set_kernel(); the dedicated N-body kernel refuses
    # programs that are not N-body-shaped (pendulum, ffnn, ...): those combinations are skipped, not failed.
    outcome = yield
    exc = outcome.excinfo
    if exc is not None and isinstance(exc[1], ValueError) and "The N-body kernel cannot run this program" in str(exc[1]):
        outcome.force_exception(pytest.skip.Exception("not an N-body-shaped program: " + str(exc[1])))
