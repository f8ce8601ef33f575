"""The drop-in Python API (`import uisrnn`) on a CUDA device: UISRNN.predict / predict_single /
parallel_predict route to libuisrnn_b200.so and reproduce the reference's golden labels."""
import numpy as np
import pytest

from helpers import inference_args, load_weights, small_cases, toy_utterances, uisrnn_from_weights

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def toy_model():
  return uisrnn_from_weights(load_weights('model_toy100.npz'), enable_cuda=True)


def test_device_and_native_library_are_used(toy_model):
  assert toy_model.device.type == 'cuda'
  xs, labs = toy_utterances()
  assert toy_model.predict(xs[0], inference_args()) == labs[0].tolist()
  native_model = toy_model._native[1]            # pylint: disable=protected-access
  stats = native_model.stats()
  assert stats['kernel_launches'] >= 3 and stats['gru_columns'] > 0   # cast + GEMM + beam kernels ran


def test_predict_list_matches_reference_on_all_toy_utterances(toy_model):
  xs, labs = toy_utterances()
  got = toy_model.predict(xs, inference_args())
  assert isinstance(got, list) and all(isinstance(g, list) for g in got)
  assert got == [l.tolist() for l in labs]
  assert all(isinstance(v, int) for v in got[0])


def test_parallel_predict_on_cuda(toy_model):
  import uisrnn
  xs, labs = toy_utterances()
  got = uisrnn.parallel_predict(toy_model, xs[:6], inference_args(), num_processes=4)
  assert got == [l.tolist() for l in labs[:6]]
  with pytest.raises(TypeError):
    uisrnn.parallel_predict(toy_model, xs[0], inference_args())


def test_exceptions_match_reference(toy_model):
  args = inference_args()
  with pytest.raises(TypeError):
    toy_model.predict(np.zeros((4, 256), np.float32), args)
  with pytest.raises(ValueError):
    toy_model.predict(np.zeros((4, 255)), args)
  with pytest.raises(ValueError):
    toy_model.predict([np.zeros((4, 256)), np.zeros(256)], args)
  with pytest.raises(TypeError):
    toy_model.predict(7, args)


def test_unsupported_configurations_raise_instead_of_falling_back():
  from uisrnn_b200 import native
  small = uisrnn_from_weights(load_weights('model_small.npz'), enable_cuda=True)
  case = [c for c in small_cases() if c['name'] == 'la2'][0]
  assert small.predict(case['x'], inference_args(5, 2, 1)) == case['labels'].tolist()   # look_ahead 2 kernel
  with pytest.raises(native.NativeError) as ei:
    small.predict(case['x'], inference_args(200, 1, 1))          # beam > 128: no kernel
  assert ei.value.code == native.UIS_ERR_UNSUPPORTED
  import uisrnn
  m, _, _ = uisrnn.parse_arguments([])
  m.rnn_depth, m.rnn_hidden_size, m.observation_dim, m.transition_bias, m.verbosity = 5, 128, 64, 0.1, 0
  deep = uisrnn.UISRNN(m)
  with pytest.raises(native.NativeError) as ei:
    deep.predict(np.random.rand(5, 64), inference_args())       # depth 5 > 4: no kernel
  assert ei.value.code == native.UIS_ERR_UNSUPPORTED
  m.rnn_hidden_size = 96                                         # no kernel instantiated for H=96
  odd = uisrnn.UISRNN(m)
  with pytest.raises(native.NativeError):
    odd.predict(np.random.rand(5, 64), inference_args())


def test_depth2_model_through_the_api():
  from helpers import depth2_cases
  model = uisrnn_from_weights(load_weights('model_small_d2.npz'), enable_cuda=True)
  for case in depth2_cases():
    args = inference_args(case['beam_size'], case['look_ahead'], case['test_iteration'])
    assert model.predict(case['x'], args) == case['labels'].tolist()


def test_cluster_table_overflow_is_retried_with_larger_tables(monkeypatch):
  from uisrnn_b200 import uisrnn as mod
  small = uisrnn_from_weights(load_weights('model_small.npz'), enable_cuda=True)
  case = [c for c in small_cases() if c['name'] == 'b10'][0]
  monkeypatch.setattr(mod, '_DEFAULT_KCAP', 1)
  assert small.predict(case['x'], inference_args(10, 1, 2)) == case['labels'].tolist()


def test_fit_on_cuda_then_native_predict_matches_cpu_decoder():
  import random
  import torch
  import uisrnn
  from uisrnn_b200.synth import synth_training_set, synth_utt
  np.random.seed(3); random.seed(3); torch.manual_seed(3)
  m, t, i = uisrnn.parse_arguments([])
  m.rnn_hidden_size, m.observation_dim, m.verbosity = 128, 64, 0
  t.train_iteration, t.batch_size, t.learning_rate = 60, 16, 2e-3
  model = uisrnn.UISRNN(m)
  assert model.device.type == 'cuda'
  seqs, ids = synth_training_set(8000, 40, n_frames=60, dim=64, n_spk=3, noise=0.08)
  model.fit(seqs, ids, t)
  tests = [synth_utt(8100 + k, n_frames=50, dim=64, n_spk=3, noise=0.08)[0] for k in range(3)]
  got = model.predict(tests, i)
  # same weights on the CPU device, decoded by beam_cpu.py
  twin = uisrnn_from_weights({k: (np.asarray(v) if not np.isscalar(v) else v)
                              for k, v in model.export_weights().items()})
  want = twin.predict(tests, i)
  assert got == want
  # parameters changed => the device twin must be rebuilt
  before = model._native[0]                      # pylint: disable=protected-access
  t.train_iteration = 2
  model.fit(seqs, ids, t)
  model.predict(tests[0], i)
  assert model._native[0] != before              # pylint: disable=protected-access


def test_edit_through_data_rebuilds_the_device_twin():
  """A sign flip of one W2 row through `.data` keeps `_version` and every |value|: predict() and score() must still
  decode the edited weights, as a fresh model that loaded them does."""
  import torch
  w = load_weights('model_toy100.npz')
  model = uisrnn_from_weights(w, enable_cuda=True)
  xs, _ = toy_utterances()
  xs = xs[:3]
  args = inference_args()
  model.predict(xs, args)  # builds the device twin
  path = [[0, 1] * (len(x) // 2) + [0] * (len(x) % 2) for x in xs]
  before_sc = model.score(xs, path)
  with torch.no_grad():
    model.rnn_model.linear_mean2.weight.data[0].neg_()
  edited = {k: (np.array(v) if not np.isscalar(v) else v) for k, v in w.items()}
  edited['w2'][0] = -edited['w2'][0]
  fresh = uisrnn_from_weights(edited, enable_cuda=True)
  want, want_sc = fresh.predict(xs, args), fresh.score(xs, path)
  assert model.predict(xs, args) == want
  assert model.score(xs, path) == want_sc
  assert want_sc != before_sc  # the edit is visible in the scores (the labels may not move)


def test_parallel_predict_thread_branch_on_two_devices(toy_model):
  """SURVEY 8(f) f3: with >= 2 visible GPUs `parallel_predict(num_processes=k)` shards the list by frame count and
  decodes every shard on its own device from its own host thread (one uis_model per device).  The caller's current
  device must be what it was, and the labels those of the reference."""
  import torch
  import uisrnn
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  xs, labs = toy_utterances()
  before = torch.cuda.current_device()
  got = uisrnn.parallel_predict(toy_model, xs, inference_args(), num_processes=torch.cuda.device_count())
  assert got == [l.tolist() for l in labs]
  assert torch.cuda.current_device() == before
  # both devices did work: device 1 now holds a context with allocations made by its uis_model
  assert torch.cuda.mem_get_info(1)[0] < torch.cuda.mem_get_info(1)[1]
