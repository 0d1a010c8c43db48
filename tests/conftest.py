import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        have = torch.cuda.is_available()
    except Exception:
        have = False
    if have:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


def pytest_collection_finish(session):
    # a GPU test that hangs (a wait nobody satisfies) must fail in minutes, not hold a GPU box until the caller's limit:
    # pytest-timeout's per-test limit, when the plugin is there and no limit was given on the command line
    if session.config.pluginmanager.hasplugin("timeout") and not session.config.getoption("timeout", None):
        for it in session.items:
            if "gpu" in it.keywords and it.get_closest_marker("timeout") is None:
                it.add_marker(pytest.mark.timeout(900))
