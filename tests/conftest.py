import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def scenes():
    """Cache of synthetic scenes (mve_b200.synth) by config name."""
    from mve_b200 import synth
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = synth.make_scene(name)
        return cache[name]
    return get


@pytest.fixture(scope="session")
def oracle_scenes(scenes):
    from oracle import oracle_py
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = oracle_py.OracleScene(scenes(name))
        return cache[name]
    return get


@pytest.fixture(scope="session")
def gpu_scenes(scenes):
    from mve_b200 import dmrecon
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = dmrecon.Scene.from_synth(scenes(name))
        return cache[name]
    return get
