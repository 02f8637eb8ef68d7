import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """`gpu`-marked tests are skipped (not errors) on a box without a CUDA device."""
    if not any("gpu" in it.keywords for it in items):
        return
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="needs a CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def tiny_scene():
    from badslam_b200.scene import config_by_name, make_scene
    return make_scene(config_by_name("tiny"))


@pytest.fixture(scope="session")
def small_scene():
    from badslam_b200.scene import config_by_name, make_scene
    return make_scene(config_by_name("small"))


@pytest.fixture(scope="session")
def cfg1_scene():
    from badslam_b200.scene import config_by_name, make_scene
    return make_scene(config_by_name("cfg1"))
