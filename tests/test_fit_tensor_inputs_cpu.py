"""fit() from tensors without a GPU: the argument checks of uis_trainer_set_corpus_device, its export, the reference's
TypeErrors for tensors on a CPU model, and the str(v) label rule of utils.concatenate_training_data."""
import ctypes
import random

import numpy as np
import pytest
import torch

from uisrnn_b200 import arguments
from uisrnn_b200 import utils


@pytest.fixture(scope='module')
def lib():
  import __graft_entry__ as ge
  ge.build()
  from uisrnn_b200 import native
  return native.load_library(), native


def test_set_corpus_device_rejects_bad_arguments_without_a_gpu(lib):
  cdll, native = lib
  bogus = ctypes.c_void_p(16)  # never dereferenced: every call below with it fails its argument checks first
  table = ctypes.c_void_p(64)

  def call(index, offsets, handle=bogus, addr=table, dtype=native.UIS_DTYPE_F32, n_rows=4, n_sub=None):
    ix, off = np.asarray(index, np.int32), np.asarray(offsets, np.int64)
    return cdll.uis_trainer_set_corpus_device(
        handle, addr, dtype, n_rows, ix.ctypes.data_as(ctypes.c_void_p), len(ix), off.ctypes.data_as(ctypes.c_void_p),
        len(off) - 1 if n_sub is None else n_sub, None)

  def fails(message, *args, **kwargs):
    return call(*args, **kwargs) == native.UIS_ERR_INVALID and message in cdll.uis_last_error()

  assert fails(b'trainer is NULL', [0, 1, 3], [0, 2, 3], handle=None)
  assert fails(b'null argument', [0, 1], [0, 2], addr=None)
  for dtype in (-1, 4, 99):
    assert fails(b'unknown dtype', [0, 1], [0, 2], dtype=dtype)
  assert fails(b'inconsistent corpus sizes', [0, 1], [0, 2], n_rows=0)
  assert fails(b'inconsistent corpus sizes', [0, 1], [0, 1])        # offsets end short of the index
  assert fails(b'inconsistent corpus sizes', [0, 1], [1, 2])        # offsets do not start at 0
  assert fails(b'inconsistent corpus sizes', [0, 1], [0, 2], n_sub=0)
  assert fails(b'out of range', [0, 4], [0, 2])
  assert fails(b'out of range', [-1, 0], [0, 2])
  assert fails(b'non-decreasing', [0, 1, 2], [0, 2, 1, 3])
  for dtype in (native.UIS_DTYPE_F16, native.UIS_DTYPE_BF16, native.UIS_DTYPE_F64):  # known dtypes reach the handle
    assert fails(b'trainer is NULL', [0, 1], [0, 2], handle=None, dtype=dtype)
  rc = cdll.uis_trainer_set_corpus_device(bogus, table, 0, 4, None, 0, None, 1, None)
  assert rc == native.UIS_ERR_INVALID and b'null argument' in cdll.uis_last_error()


def test_binding_exports_the_entry_point(lib):
  cdll, native = lib
  assert 'uis_trainer_set_corpus_device' in native.EXPORTS
  assert hasattr(cdll, 'uis_trainer_set_corpus_device')
  assert hasattr(native.NativeTrainer, 'set_corpus_device')
  assert (native.UIS_DTYPE_F32, native.UIS_DTYPE_F16, native.UIS_DTYPE_BF16, native.UIS_DTYPE_F64) == (0, 1, 2, 3)


def _cpu_model():
  from uisrnn_b200 import uisrnn
  model_args, _, _ = arguments.parse_arguments([])
  model_args.enable_cuda = False
  model_args.observation_dim = 4
  model_args.rnn_hidden_size = 8
  return uisrnn.UISRNN(model_args)


def test_cpu_model_raises_the_reference_type_errors():
  model = _cpu_model()
  _, training_args, _ = arguments.parse_arguments([])
  training_args.train_iteration = 1
  x = torch.zeros(6, 4, dtype=torch.float64)
  labels = ['a'] * 6
  with pytest.raises(TypeError, match='train_sequences must be a list or numpy.ndarray'):
    model.fit(x, labels, training_args)
  with pytest.raises(TypeError, match='train_sequence should be a numpy array of float type.'):
    model.fit([x], [labels], training_args)
  with pytest.raises(TypeError, match='train_sequence should be a numpy array of float type.'):
    model.fit([x, x.float()], [labels, labels], training_args)
  with pytest.raises(TypeError, match='train_sequence should be a numpy array of float type.'):
    model.fit_concatenated(x, np.array(labels), training_args)
  assert model.transition_bias is None  # nothing was estimated before the error


def test_ndarray_sequences_keep_the_reference_label_rules():
  """Label tensors are converted on the tensor route only: with ndarray sequences, a CPU model and the helper raise
  the reference's TypeError for them, as before."""
  model = _cpu_model()
  _, training_args, _ = arguments.parse_arguments([])
  training_args.train_iteration = 1
  xs = [np.zeros((6, 4)) for _ in range(3)]
  labels = [torch.tensor([0, 0, 1, 1, 2, 2]) for _ in range(3)]
  with pytest.raises(TypeError, match='Elements of train_cluster_ids must be list or numpy.ndarray'):
    model.fit(xs, labels, training_args)
  for uniqueness in (True, False):
    with pytest.raises(TypeError, match='Elements of train_cluster_ids must be list or numpy.ndarray'):
      utils.concatenate_training_data(xs, labels, uniqueness, True)


def test_host_labels_reads_integer_tensors_as_strings():
  ids = torch.tensor([[7, 0], [-3, 0], [7, 0], [2 ** 40, 0]], dtype=torch.int64)[:, 0]  # strided
  out = utils.host_labels([ids, ['x', 'y'], torch.tensor([1, 1], dtype=torch.int8), np.array(['p'])])
  assert out[0] == ['7', '-3', '7', str(2 ** 40)]
  assert out[1] == ['x', 'y'] and out[2] == ['1', '1'] and out[3].tolist() == ['p']
  big = torch.tensor([[2 ** 64 - 1, 0], [5, 0], [2 ** 63, 0]], dtype=torch.uint64)[:, 0]  # no wrap-around
  assert utils.host_labels([big, torch.tensor([7], dtype=torch.uint32)]) == [
      [str(2 ** 64 - 1), '5', str(2 ** 63)], ['7']]
  plain = [['a'], np.array(['b'])]
  assert utils.host_labels(plain) is plain
  with pytest.raises(TypeError, match='integer dtype'):
    utils.host_labels([torch.zeros(3)])
  with pytest.raises(TypeError, match='integer dtype'):
    utils.host_labels([torch.zeros(3, dtype=torch.bool)])
  with pytest.raises(ValueError, match='1-D'):
    utils.host_labels([torch.zeros(3, 1, dtype=torch.int32)])


@pytest.mark.parametrize('uniqueness', [True, False])
def test_concatenate_training_data_str_rule_and_shuffle(uniqueness):
  """Tensors with integer label tensors give the shuffled tensor list and the labels that the same values as ndarrays
  with str(v) labels give, after the same `random` calls."""
  rng = np.random.default_rng(3)
  lengths = [5, 0, 3, 7, 2]
  arrays = [rng.standard_normal((n, 4)) for n in lengths]
  ints = [rng.integers(-4, 4, n) for n in lengths]
  tensors = [torch.from_numpy(a).float() for a in arrays]
  label_tensors = [torch.from_numpy(v).to(torch.int32) for v in ints]
  label_tensors[2] = [str(v) for v in ints[2]]  # a host label sequence among the tensors
  random.seed(11)
  want_x, want_ids = utils.concatenate_training_data(arrays, [[str(v) for v in v_] for v_ in ints], uniqueness, True)
  want_state = random.getstate()
  random.seed(11)
  got_x, got_ids = utils.concatenate_training_data(tensors, label_tensors, uniqueness, True)
  assert random.getstate() == want_state
  assert got_ids == want_ids
  assert isinstance(got_x, list) and all(isinstance(t, torch.Tensor) for t in got_x)
  assert np.array_equal(torch.cat(got_x).double().numpy(), want_x.astype(np.float32).astype(np.float64))
  by_id = {id(t): i for i, t in enumerate(tensors)}
  order = [by_id[id(t)] for t in got_x]  # the tensors themselves, not copies, in the shuffled order
  assert sorted(order) == list(range(len(tensors)))
  assert np.array_equal(torch.cat(got_x).numpy(), np.concatenate([arrays[i] for i in order]).astype(np.float32))


def test_concatenate_training_data_checks_tensor_lists():
  with pytest.raises(ValueError, match='same length'):
    utils.concatenate_training_data([torch.zeros(3, 2)], [torch.tensor([1, 2])], False, False)
  with pytest.raises(ValueError, match='consistent observation dimension'):
    utils.concatenate_training_data([torch.zeros(1, 2), torch.zeros(1, 3)], [[1], [1]], False, False)
