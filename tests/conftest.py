import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


def pytest_addoption(parser):
    parser.addoption("--cuemu", action="store_true", default=False,
                     help="run the tests marked `gpu` on the CPU under the cuemu fiber emulator (tests/cuemu): "
                          "`pytest tests -m gpu --cuemu`.  Tests that need CUDA graphs or 2 GPUs fail or skip.")


import pytest  # noqa: E402


@pytest.fixture(autouse=True)
def _cuemu_for_gpu_tests(request, monkeypatch):
    if request.config.getoption("--cuemu") and request.node.get_closest_marker("gpu") is not None:
        from tests.cuemu import harness
        harness.set_order("fwd")
        harness.emulated_device(monkeypatch)
        from mmssl_b200 import evaluate
        import functools
        monkeypatch.setattr(evaluate, "Evaluator", functools.partial(evaluate.Evaluator, device="cpu"))
    yield
