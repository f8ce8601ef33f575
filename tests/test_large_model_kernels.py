"""The (hidden 1024, dim 512) kernel shape decodes stacked GRUs and look-ahead trees: the built library must carry the
sm_90a code of those instantiations (no GPU needed)."""
import os
import shutil
import subprocess

import pytest


def test_sass_has_the_deep_and_look_ahead_1024x512_kernels():
  tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
  if not os.path.exists(tool):
    pytest.skip('cuobjdump not available')
  from uisrnn_b200 import native
  sass = subprocess.run([tool, '-sass', native.LIB_PATH], capture_output=True, text=True).stdout
  for name in ('uis_beam_kernelILi1024ELi512ELb1E',        # look_ahead 1, rnn_depth 2..4
               'uis_beam_tree_kernelILi1024ELi512ELb0E',   # look_ahead >= 2, rnn_depth 1
               'uis_beam_tree_kernelILi1024ELi512ELb1E'):  # look_ahead >= 2, rnn_depth 2..4
    start = sass.find(name)
    assert start >= 0, name + ' is not in the library'
    body = sass[start:sass.find('Function :', start + len(name))]
    assert 'sm_90a' in sass and 'FFMA' in body and 'UBLKCP' in body, name
