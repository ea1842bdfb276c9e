import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as o
    o.build()
    return o


@pytest.fixture(scope="session")
def pair_scene():
    from voxgraph_b200 import synth
    return synth.make_pair_scene(seed=1, n_points=1000)


@pytest.fixture(scope="session")
def small_scene():
    """Scaled-down config 2: 6 submaps, 2k points each."""
    from voxgraph_b200 import synth
    return synth.make_scene(seed=2, n_submaps=6, n_points=2000, radius=8.0,
                            size_xy=(48.0, 32.0), n_clutter=80, n_walls=6)
