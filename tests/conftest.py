import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `pytest -m gpu`)")


# Sokoban reads Boxoban level files (scenario_sokoban.cpp:39-81); the dataset is not available offline, so the tests point
# both sides at a small synthetic set in the same text format
os.environ.setdefault("BOXOBAN_LEVELS", os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "boxoban"))


@pytest.fixture(scope="session")
def built():
    """make sure the in-tree native libraries exist (nvcc cross-compiles without a GPU)"""
    from megaverse_b200 import _build

    _build.build_all()
    import orc

    orc.lib()
    return True
