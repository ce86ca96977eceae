import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
  config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')


def load_golden(name):
  z = np.load(os.path.join(GOLDEN_DIR, name + '.npz'))
  d = {k: z[k] for k in z.files}
  d['meta'] = json.loads(bytes(d['meta']).decode())
  return d


@pytest.fixture(scope='session')
def golden():
  return load_golden
