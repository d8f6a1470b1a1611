import os
import sys
from pathlib import Path

import numpy
import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs an H100 (sm_90a)')


def _has_gpu() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason='no CUDA device in this container')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope='session')
def engine():
    from realtime_yukarin_b200.engine import default_engine
    return default_engine()


@pytest.fixture(scope='session')
def small_models(tmp_path_factory):
    """Seeded synthetic model files with narrow U-Nets (base 16): fast for the CPU oracle."""
    from realtime_yukarin_b200.synthetic import write_synthetic_models
    d = tmp_path_factory.mktemp('models_small')
    return write_synthetic_models(d, seed=3, base1=16, base2=16)


@pytest.fixture(scope='session')
def full_models(tmp_path_factory):
    """Full-width synthetic models (base 64: stage 1 13.6 M, stage 2 54.4 M parameters)."""
    from realtime_yukarin_b200.synthetic import write_synthetic_models
    d = tmp_path_factory.mktemp('models_full')
    return write_synthetic_models(d, seed=0)
