"""Look-ahead trees that outgrow shared memory are decoded by the spill instantiations of the tree kernel (arena in
device memory): the built library must carry their sm_90a code for every kernel shape and rnn_depth (no GPU needed)."""
import os
import shutil
import subprocess

import pytest


def test_sass_has_the_tree_spill_kernels():
  tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
  if not os.path.exists(tool):
    pytest.skip('cuobjdump not available')
  from uisrnn_b200 import native
  sass = subprocess.run([tool, '-sass', native.LIB_PATH], capture_output=True, text=True).stdout
  assert 'sm_90a' in sass
  for H, D in ((128, 64), (256, 128), (512, 256), (1024, 512)):
    for deep in (0, 1):
      name = 'uis_beam_tree_kernelILi%dELi%dELb%dELb1E' % (H, D, deep)  # <H, D, DEEP, SPILL = true>
      start = sass.find(name)
      assert start >= 0, name + ' is not in the library'
      body = sass[start:sass.find('Function :', start + len(name))]
      # FFMA weight passes fed by the bulk-copy ring; the radix select's warp-aggregated histogram (MATCH)
      assert 'FFMA' in body and 'UBLKCP' in body and 'MATCH' in body, name
