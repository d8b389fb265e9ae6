import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on an H100 with -m gpu)')


@pytest.fixture(scope='session')
def golden():
    arrays = np.load(os.path.join(GOLDEN_DIR, 'ref_golden.npz'))
    with open(os.path.join(GOLDEN_DIR, 'ref_golden.json')) as f:
        meta = json.load(f)
    return arrays, meta


def golden_configs():
    """The encoder configurations the fixtures were generated with (kept in make_golden.py)."""
    sys.path.insert(0, GOLDEN_DIR)
    import importlib.util
    src = open(os.path.join(GOLDEN_DIR, 'make_golden.py')).read()
    # CONFIGS is a pure literal apart from two imported aspect-ratio lists; evaluate it without
    # importing the reference.
    from oracle.model import SSD300_AR, SSD512_AR
    start = src.index('CONFIGS = {')
    end = src.index('\n}\n', start) + 3
    ns = {'SSD300_AR': SSD300_AR, 'SSD512_AR': SSD512_AR}
    exec(src[start:end], ns)
    return ns['CONFIGS']


@pytest.fixture(scope='session')
def configs():
    return golden_configs()
