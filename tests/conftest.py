"""pytest configuration: registers the `gpu` marker and puts the repo root on sys.path."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
  config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on an H100)')


def pytest_collection_modifyitems(config, items):
  """`gpu` tests need a CUDA device AND the built library; elsewhere they are skipped, not failed."""
  del config
  reason = None
  try:
    import torch
    if not torch.cuda.is_available():
      reason = 'no CUDA device'
  except Exception as err:  # pylint: disable=broad-except
    reason = 'torch unavailable: %s' % err
  if reason is None and not os.path.exists(os.path.join(ROOT, 'uisrnn_b200', 'libuisrnn_b200.so')):
    try:
      import __graft_entry__ as ge
      ge.build()
    except Exception as err:  # pylint: disable=broad-except
      reason = 'libuisrnn_b200.so missing and not buildable: %s' % err
  if reason:
    skip = pytest.mark.skip(reason=reason)
    for item in items:
      if 'gpu' in item.keywords:
        item.add_marker(skip)


@pytest.fixture(scope='session')
def golden_dir():
  return GOLDEN
