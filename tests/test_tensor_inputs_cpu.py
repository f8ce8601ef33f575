"""Tensor inputs without a GPU: the argument checks of uis_score_device_ids, the rules a list of tensors must follow,
and the reference's TypeError for tensors on a CPU model."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import inference_args, load_weights, uisrnn_from_weights


@pytest.fixture(scope='module')
def lib():
  import __graft_entry__ as ge
  ge.build()
  from uisrnn_b200 import native
  return native.load_library(), native


def test_score_device_ids_rejects_bad_arguments_without_a_gpu(lib):
  cdll, native = lib
  buf = ctypes.c_void_p(16)  # never dereferenced: every call below fails its argument checks first
  alpha, bias = (ctypes.c_double * 1)(1.0), (ctypes.c_double * 1)(0.5)
  dp = native.DecodeParams(1, alpha, bias)

  def call(offsets, x=buf, ids=buf, scores=buf):
    off = np.asarray(offsets, np.int64)
    return cdll.uis_score_device_ids(None, x, off.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), len(off) - 1, ids,
                                     scores, None, None, None, ctypes.byref(dp))

  assert call([0, 3]) == native.UIS_ERR_INVALID and b'model is NULL' in cdll.uis_last_error()
  assert call([0, 3], scores=None) == native.UIS_ERR_INVALID and b'null argument' in cdll.uis_last_error()
  assert call([0, 3], x=None) == native.UIS_ERR_INVALID and b'null device buffer' in cdll.uis_last_error()
  assert call([0, 3], ids=None) == native.UIS_ERR_INVALID and b'null device buffer' in cdll.uis_last_error()
  assert call([0, 3, 2]) == native.UIS_ERR_INVALID and b'not monotone' in cdll.uis_last_error()
  assert call([1, 3]) == native.UIS_ERR_INVALID and b'frame_offsets[0]' in cdll.uis_last_error()
  assert call([0, 3], x=ctypes.c_void_p(20)) == native.UIS_ERR_INVALID and b'aligned' in cdll.uis_last_error()
  assert call([0, 3], ids=ctypes.c_void_p(20)) == native.UIS_ERR_INVALID and b'aligned' in cdll.uis_last_error()
  rc = cdll.uis_score_device_ids(None, buf, None, 1, buf, buf, None, None, None, ctypes.byref(dp))
  assert rc == native.UIS_ERR_INVALID and b'null argument' in cdll.uis_last_error()
  # no rows: nothing to read, so only the handle is missing
  assert call([0, 0], x=None, ids=None) == native.UIS_ERR_INVALID and b'model is NULL' in cdll.uis_last_error()


def test_binding_exports_the_entry_point(lib):
  _, native = lib
  assert 'uis_score_device_ids' in native.EXPORTS
  assert hasattr(native.NativeModel, 'score_device_ids')


@pytest.fixture(scope='module')
def cpu_model():
  return uisrnn_from_weights(load_weights('model_small.npz'))


def test_cpu_model_raises_the_reference_type_error(cpu_model):
  args = inference_args(beam_size=2, test_iteration=1)
  x = torch.zeros(5, cpu_model.observation_dim, dtype=torch.float64)
  with pytest.raises(TypeError, match='test_sequences should be either a list or numpy array.'):
    cpu_model.predict(x, args)
  with pytest.raises(TypeError, match='test_sequence should be a numpy array of float type.'):
    cpu_model.predict_single(x, args)
  with pytest.raises(TypeError, match='test_sequence should be a numpy array of float type.'):
    cpu_model.predict([x], args)
  with pytest.raises(TypeError, match='test_sequences should be either a list or numpy array.'):
    cpu_model.score(x, [0] * 5)
  with pytest.raises(TypeError, match='test_sequence should be a numpy array of float type.'):
    cpu_model.score([x], [[0] * 5])


def test_tensor_list_rules():
  from uisrnn_b200.uisrnn import _tensor_sequences
  dev = torch.device('cpu')
  a, b = torch.zeros(4, 3), torch.zeros(2, 3)
  assert _tensor_sequences([a, b], 3, dev) is True
  assert _tensor_sequences([np.zeros((4, 3))], 3, dev) is False
  assert _tensor_sequences([], 3, dev) is False
  with pytest.raises(TypeError, match='not a mix'):
    _tensor_sequences([a, np.zeros((2, 3))], 3, dev)
  with pytest.raises(TypeError, match='not a mix'):
    _tensor_sequences([np.zeros((2, 3)), a], 3, dev)
  with pytest.raises(TypeError, match='share a dtype'):
    _tensor_sequences([a, b.double()], 3, dev)
  with pytest.raises(TypeError, match='share a dtype'):
    _tensor_sequences([a.half(), b.bfloat16()], 3, dev)
  with pytest.raises(TypeError, match='float32, float16, bfloat16 or float64'):
    _tensor_sequences([a.int()], 3, dev)
  for dtype in (torch.float32, torch.float16, torch.bfloat16, torch.float64):
    assert _tensor_sequences([a.to(dtype), b.to(dtype)], 3, dev)
  assert _tensor_sequences([torch.zeros(3, 4).t()], 3, dev)  # strided
  with pytest.raises(ValueError, match='2-dim'):
    _tensor_sequences([torch.zeros(3)], 3, dev)
  with pytest.raises(ValueError, match='observation_dim'):
    _tensor_sequences([torch.zeros(2, 4)], 3, dev)
  with pytest.raises(ValueError, match="model's device"):
    _tensor_sequences([a], 3, torch.device('cuda', 0))


def test_device_rows_and_ids_on_the_host():
  """The host-side pieces of the conversion: one fp32 buffer (the caller's own when it already is one), float64 rounded
  to nearest, offsets, and label sequences renamed before upload."""
  from uisrnn_b200.uisrnn import _device_ids, _device_rows
  a = torch.arange(12, dtype=torch.float32).reshape(4, 3)
  x, off = _device_rows([a])
  assert x.data_ptr() == a.data_ptr() and off.tolist() == [0, 4]
  v = torch.tensor([[1 + 2.0 ** -30, 3.0, 1 - 2.0 ** -27]], dtype=torch.float64)
  x, off = _device_rows([a.double(), v, torch.zeros(0, 3, dtype=torch.float64)])
  assert x.dtype == torch.float32 and x.is_contiguous() and off.tolist() == [0, 4, 5, 5]
  assert np.array_equal(x.numpy(), np.concatenate([a.numpy(), v.numpy().astype(np.float32)]))
  w = torch.zeros(3, 5).t()
  x, _ = _device_rows([w.requires_grad_()])
  assert x.is_contiguous() and not x.requires_grad
  ids = _device_ids([['b', 'a', 'b'], torch.tensor([7, -1], dtype=torch.int16)], [3, 2], torch.device('cpu'))
  assert ids.dtype == torch.int64 and ids.tolist() == [0, 1, 0, 7, -1]
  with pytest.raises(ValueError, match='2 labels for 3 frames'):
    _device_ids([[0, 1]], [3], torch.device('cpu'))
  with pytest.raises(TypeError, match='integer dtype'):
    _device_ids([torch.zeros(3)], [3], torch.device('cpu'))


def test_conversion_copies_strided_ids_and_misaligned_rows():
  """A strided int64 label tensor (which .to(int64) hands back as itself) is made contiguous, also for one utterance;
  a contiguous fp32 view off a 16-byte boundary is copied into a fresh (aligned) buffer instead of passed through."""
  from uisrnn_b200.uisrnn import _device_ids, _device_rows
  base = torch.arange(20, dtype=torch.int64).reshape(10, 2)
  for ids in (base[:, 1], base.reshape(-1)[::2], torch.tensor([5]).expand(10)):
    got = _device_ids([ids], [10], torch.device('cpu'))
    assert got.is_contiguous() and got.tolist() == ids.tolist()
  flat = torch.arange(1 + 4 * 8, dtype=torch.float32)
  shifted = flat[1:].view(4, 8)
  assert shifted.is_contiguous() and shifted.data_ptr() % 16 != 0
  x, _ = _device_rows([shifted])
  assert x.data_ptr() % 16 == 0 and x.data_ptr() != shifted.data_ptr() and torch.equal(x, shifted)
