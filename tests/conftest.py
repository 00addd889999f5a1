import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'oracle')):
  if p not in sys.path:
    sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
  config.addinivalue_line('markers', 'gpu: needs a CUDA device (H100); run with -m gpu on a GPU machine')


@pytest.fixture(scope='session')
def golden_dir():
  return GOLDEN


@pytest.fixture(scope='session')
def built_lib():
  """Path of libctb200.so, building it (nvcc, sm_90a) if needed."""
  from centertrack_b200 import _lib
  return _lib.build()
