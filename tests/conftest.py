import os
import sys

import pytest

# tests need the grounder's shapes, not RoBERTa's checkpoint (no network): opt in to the random-init text encoder
os.environ.setdefault('ESB200_TEXT_RANDOM_INIT', '1')

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100: run with `-m gpu`)')


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(autouse=True)
def _restore_collector():
    """engine.OptimWrapper takes the cyclic collector over for the lifetime of a training job (gc_interval); a test session
    builds many short-lived models, so every test hands the interpreter's automatic collection back and frees what it left."""
    import gc
    yield
    gc.enable()
    gc.collect()
