import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a GPU machine)")
    config.addinivalue_line("markers", "reference: needs the read-only reference checkout at /root/reference")


def pytest_collection_modifyitems(config, items):
    """A hung kernel must fail one test, not the GPU box: every test gets a wall-clock limit (pytest-timeout, when installed)."""
    if not config.pluginmanager.hasplugin("timeout"):
        return
    for it in items:
        if it.get_closest_marker("timeout") is None:
            # GPU tests: method="thread" (the watchdog ends the process) — a signal cannot interrupt a blocked cudaStreamSynchronize
            if it.get_closest_marker("gpu"):
                it.add_marker(pytest.mark.timeout(600, method="thread"))
            else:
                it.add_marker(pytest.mark.timeout(300))
