import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
  sys.path.insert(0, REPO)

GOLDEN = os.path.join(REPO, 'tests', 'golden')


def pytest_configure(config):
  config.addinivalue_line('markers', 'slow: takes more than a few seconds on CPU')
  config.addinivalue_line('markers', 'gpu: test needs a CUDA device (run with -m gpu on an H100)')


def pytest_collection_modifyitems(config, items):
  import torch
  if torch.cuda.is_available():
    return
  skip = pytest.mark.skip(reason='no CUDA device')
  for item in items:
    if 'gpu' in item.keywords:
      item.add_marker(skip)


@pytest.fixture(scope='session')
def golden_dir():
  return GOLDEN
