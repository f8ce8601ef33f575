"""The C-ABI shared library: builds for sm_90a without a GPU, loads, and exports every symbol
include/uisrnn_b200.h declares.  No compute calls here (CPU only)."""
import ctypes
import os
import re

import pytest

from helpers import ROOT


@pytest.fixture(scope='module')
def lib():
  import __graft_entry__ as ge
  ge.build()
  from uisrnn_b200 import native
  return native.load_library(), native


def test_header_symbols_are_exported(lib):
  cdll, native = lib
  header = open(os.path.join(ROOT, 'include', 'uisrnn_b200.h')).read()
  body = re.sub(r'/\*.*?\*/', '', header, flags=re.S)
  declared = set(re.findall(r'\b(uis_[a-z_]+)\s*\(', body))
  assert declared == set(native.EXPORTS), declared ^ set(native.EXPORTS)
  for name in declared:
    assert getattr(cdll, name) is not None


def native_version():
  header = open(os.path.join(ROOT, 'include', 'uisrnn_b200.h')).read()
  return int(re.search(r'#define UIS_ABI_VERSION (\d+)', header).group(1))


def test_version_and_error_string(lib):
  cdll, native = lib
  assert native.UIS_ABI_VERSION == native_version()
  assert cdll.uis_version() == native_version()
  assert isinstance(cdll.uis_last_error(), bytes)


def test_struct_layouts_match_header(lib):
  _, native = lib
  assert ctypes.sizeof(native.PredictOpts) == 8 * 4
  assert ctypes.sizeof(native.DebugTaps) == 8 + 8 * 8
  assert ctypes.sizeof(native.Stats) == 7 * 8 + 2 * 4 + 2 * 4 + 4 * 4 + 10 * 8 + 4 * 8 + 6 * 4  # + host-path timings (ABI 4)
  assert ctypes.sizeof(native.TrainHParams) == 6 * 4 + 2 * 4 + 8  # + rnn_depth, rnn_dropout, dropout_seed (ABI 4)


def test_invalid_arguments_are_rejected_without_a_gpu(lib):
  cdll, native = lib
  handle = ctypes.c_void_p()
  rc = cdll.uis_model_create(ctypes.byref(handle), 0, 256, 512, 1, *([None] * 10), 0.1, 1.0)
  assert rc == native.UIS_ERR_INVALID and b'NULL' in cdll.uis_last_error()
  assert cdll.uis_model_destroy(None) == 0


def test_sass_uses_tma_and_register_rebalancing():
  """The hot kernel must contain TMA bulk copies (UBLKCP) and mbarrier ops (SYNCS)."""
  import shutil
  import subprocess
  tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
  if not os.path.exists(tool):
    pytest.skip('cuobjdump not available')
  from uisrnn_b200 import native
  sass = subprocess.run([tool, '-sass', native.LIB_PATH], capture_output=True, text=True).stdout
  assert 'UBLKCP' in sass and 'SYNCS' in sass
  # register re-balancing of the warp-specialised CTA, and the cluster (latency) mode: cluster barrier at start-up,
  # remote mbarrier arrives (the .RED form) for the distributed-shared-memory exchange
  assert 'USETMAXREG' in sass and 'UCGABAR_ARV' in sass and 'SYNCS.ARRIVE.TRANS64.RED' in sass


def test_sass_uses_wgmma_and_tensor_map_tma():
  """The tensor-core engine must be the real thing: warpgroup MMAs (HGMMA, with the WARPGROUP fences and waits around
  them) and tensor-map TMA (UTMALDG) inside the uis_beam_kernel<.., columns> instantiations."""
  import shutil
  import subprocess
  tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
  if not os.path.exists(tool):
    pytest.skip('cuobjdump not available')
  from uisrnn_b200 import native
  sass = subprocess.run([tool, '-sass', native.LIB_PATH], capture_output=True, text=True).stdout
  start = sass.find('uis_beam_kernelILi512ELi256ELb0ELi0ELi48EE')
  assert start >= 0, 'tensor-core instantiation missing'
  end = sass.find('Function :', start + 10)
  body = sass[start:end if end > 0 else len(sass)]
  for mnemonic in ('HGMMA.64x96x16.F32', 'WARPGROUP', 'UTMALDG', 'SYNCS'):
    assert mnemonic in body, mnemonic
