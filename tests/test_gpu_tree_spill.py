"""Look-ahead beam steps whose candidate tree outgrows shared memory are decoded by the spill kernel, from a
device-memory arena, by the same algorithm.  Every case is compared with the CPU oracle (or the reference goldens):
labels identical, per-step scores within 1e-5 relative, best hidden states / running means within 1e-5 absolute.

The natural-spill cases also check that the same call with UISRNN_B200_TREE_SPILL=0 (the shared-memory kernel
alone) raises UIS_ERR_CAPACITY, so that they exercise the spill kernel; UISRNN_B200_TREE_SPILL=force sends every
utterance of a look-ahead call to it."""
import random

import numpy as np
import pytest

from helpers import compare_trace, load_weights, oracle_model, rel_err, small_cases, uis_oracle
from test_gpu_large_models import _cached, check_against_oracle, utterances
from test_gpu_parity import _random_weights

pytestmark = pytest.mark.gpu

SCORE_RTOL = 1e-5
STATE_ATOL = 1e-5


@pytest.fixture(scope='module')
def native():
  from uisrnn_b200 import native as nat
  nat.load_library()
  return nat


@pytest.fixture(scope='module')
def toy_model(native):
  return native.NativeModel(load_weights('model_toy100.npz'))


def raises_capacity_without_spill(native, monkeypatch, call):
  monkeypatch.setenv('UISRNN_B200_TREE_SPILL', '0')
  try:
    with pytest.raises(native.NativeError) as ei:
      call()
    assert ei.value.code == native.UIS_ERR_CAPACITY
    assert 'on-chip' in str(ei.value)
  finally:
    monkeypatch.delenv('UISRNN_B200_TREE_SPILL')


# ---- 1. natural spill -------------------------------------------------------------------------------------------

def test_natural_spill_at_1024x512_depth2_look_ahead3(native, monkeypatch):
  """beam 10 on 30 frames: a step's tree holds more than the about 350 nodes that fit on chip at this shape."""
  _, model, _ = _cached(native, 1024, 512, 2)
  xs = utterances(512, 720, (30, 7))
  raises_capacity_without_spill(native, monkeypatch,
                                lambda: model.predict(xs, beam_size=10, look_ahead=3, test_iteration=1))
  check_against_oracle(native, 1024, 512, 2, 10, 3, 1, (30, 7), seed=720)


def test_natural_spill_toy_model_beam30_look_ahead3(native, monkeypatch, toy_model):
  from uisrnn_b200.synth import synth_utt
  om = oracle_model('model_toy100.npz')
  x = synth_utt(1234, n_frames=40)[0]
  call = lambda: toy_model.predict([x], beam_size=30, look_ahead=3, test_iteration=1, trace_utt=0)
  raises_capacity_without_spill(native, monkeypatch, call)
  labs, dbg = call()
  rec = {}
  want = uis_oracle.predict_single(om, x, beam_size=30, look_ahead=3, test_iteration=1, record=rec)
  assert labs[0].tolist() == want and len(set(want)) >= 3
  compare_trace(dbg['win'], dbg['score'], dbg['off'], rec['win'], rec['score'], rec['off'], rtol=SCORE_RTOL)
  assert np.max(np.abs(dbg['best_hidden'] - rec['final_hidden'])) < STATE_ATOL
  assert np.max(np.abs(dbg['best_mean'] - rec['final_mean'])) < STATE_ATOL


# ---- 2. forced spill: the look-ahead cases pinned elsewhere -----------------------------------------------------

@pytest.fixture
def forced(monkeypatch):
  monkeypatch.setenv('UISRNN_B200_TREE_SPILL', 'force')


def test_forced_config3_toy_model(forced, toy_model):
  from uisrnn_b200.synth import synth_utt
  om = oracle_model('model_toy100.npz')
  x = synth_utt(1234, n_frames=24)[0]
  got = toy_model.predict([x], beam_size=30, look_ahead=2, test_iteration=2)[0]
  assert toy_model.stats()['kernel_launches'] == 3  # cast, projection and the spill kernel alone
  assert got.tolist() == uis_oracle.predict_single(om, x, beam_size=30, look_ahead=2, test_iteration=2)


@pytest.mark.parametrize('fixture,weights', [('small_cases.npz', 'model_small.npz'),
                                             ('depth2_cases.npz', 'model_small_d2.npz')])
def test_forced_look_ahead_golden_cases(forced, native, fixture, weights):
  model = native.NativeModel(load_weights(weights))
  cases = [c for c in small_cases(fixture) if c['look_ahead'] > 1]
  assert cases
  for case in cases:
    labs, dbg = model.predict([case['x']], beam_size=case['beam_size'], look_ahead=case['look_ahead'],
                              test_iteration=case['test_iteration'], trace_utt=0)
    assert labs[0].tolist() == case['labels'].tolist(), case['name']
    compare_trace(dbg['win'], dbg['score'], dbg['off'], case['win'], case['score'], case['off'], rtol=SCORE_RTOL)
    nb = len(case['final_scores'])
    assert rel_err(dbg['final_scores'][0][:nb], case['final_scores']) < SCORE_RTOL
    assert np.max(np.abs(dbg['best_hidden'] - case['final_hidden'])) < STATE_ATOL
    assert np.max(np.abs(dbg['best_mean'] - case['final_mean'])) < STATE_ATOL


def test_forced_padded_600x300_depth2(forced, native):
  check_against_oracle(native, 600, 300, 2, 10, 2, 1, (30, 9), seed=300 + 600)


def test_forced_1024x512_depth2_look_ahead2_kcap32(forced, native):
  check_against_oracle(native, 1024, 512, 2, 10, 2, 1, (60, 7), seed=710, kcap=32)


@pytest.mark.parametrize('H,D', [(256, 128), (128, 64), (512, 256)])
def test_forced_random_models_all_kernel_shapes(forced, native, H, D):
  """The random models of test_random_models_all_kernel_shapes_match_oracle at (beam 4, look_ahead 2), every
  utterance decoded from the arena, with no exception branch."""
  w = _random_weights(H, D, seed=H + D)
  model = native.NativeModel(w)
  om = uis_oracle.OracleModel(w)
  rng = np.random.default_rng(7)
  xs = [rng.standard_normal((n, D)) * 0.3 for n in (17, 5, 26)]
  got = model.predict(xs, beam_size=4, look_ahead=2, test_iteration=2, kcap=48)
  for x, o in zip(xs, got):
    assert o.tolist() == uis_oracle.predict_single(om, x, beam_size=4, look_ahead=2, test_iteration=2)


# ---- 3. mixed batch ---------------------------------------------------------------------------------------------

def test_mixed_batch_is_independent_of_batching(native, monkeypatch):
  """Long utterances spill at look_ahead 3 / beam 10, the short ones fit on chip."""
  _, model, om = _cached(native, 1024, 512, 2)
  xs = utterances(512, 730, (30, 4, 26, 3, 5))
  raises_capacity_without_spill(native, monkeypatch, lambda: model.predict(xs[:1], beam_size=10, look_ahead=3,
                                                                            test_iteration=1))
  model.predict(xs[3:4], beam_size=10, look_ahead=3, test_iteration=1)  # fits: no error without the spill kernel
  monkeypatch.setenv('UISRNN_B200_TREE_SPILL', '0')
  model.predict(xs[3:5], beam_size=10, look_ahead=3, test_iteration=1)
  monkeypatch.delenv('UISRNN_B200_TREE_SPILL')
  together = model.predict(xs, beam_size=10, look_ahead=3, test_iteration=1)
  for n_ctas in (1, 2):
    got = model.predict(xs, beam_size=10, look_ahead=3, test_iteration=1, n_ctas=n_ctas)
    assert all(a.tolist() == b.tolist() for a, b in zip(got, together)), n_ctas
  for i, x in enumerate(xs):
    assert model.predict([x], beam_size=10, look_ahead=3, test_iteration=1)[0].tolist() == together[i].tolist()
    assert together[i].tolist() == uis_oracle.predict_single(om, x, beam_size=10, look_ahead=3, test_iteration=1)


# ---- 4. device path ---------------------------------------------------------------------------------------------

def test_device_path_spills(native, monkeypatch):
  import torch
  _, model, om = _cached(native, 1024, 512, 2)
  xs = utterances(512, 720, (30, 7))
  x = torch.from_numpy(np.concatenate(xs).astype(np.float32)).cuda()
  labels = torch.full((x.shape[0],), -7, dtype=torch.int32, device='cuda')
  off = np.concatenate([[0], np.cumsum([len(v) for v in xs])]).astype(np.int64)
  monkeypatch.setenv('UISRNN_B200_TREE_SPILL', '0')
  model.predict_device(x.data_ptr(), off, labels.data_ptr(), beam_size=10, look_ahead=3, test_iteration=1)
  with pytest.raises(native.NativeError) as ei:
    model.stats()
  assert ei.value.code == native.UIS_ERR_CAPACITY
  monkeypatch.delenv('UISRNN_B200_TREE_SPILL')
  model.predict_device(x.data_ptr(), off, labels.data_ptr(), beam_size=10, look_ahead=3, test_iteration=1)
  st = model.stats()  # errors surface here; none
  assert st['kernel_launches'] == 3
  got = labels.cpu().numpy()
  for i, v in enumerate(xs):
    assert got[off[i]:off[i + 1]].tolist() == uis_oracle.predict_single(om, v, beam_size=10, look_ahead=3,
                                                                         test_iteration=1)


# ---- 5. public API ----------------------------------------------------------------------------------------------

def test_fit_then_predict_512d_depth2_look_ahead3_through_the_api(native, monkeypatch):
  import torch
  import uisrnn
  from uisrnn_b200.synth import synth_training_set, synth_utt
  np.random.seed(7); random.seed(7); torch.manual_seed(7)
  m, t, i = uisrnn.parse_arguments([])
  m.observation_dim, m.rnn_hidden_size, m.rnn_depth, m.verbosity = 512, 512, 2, 0
  m.sigma2 = 0.003
  model = uisrnn.UISRNN(m)
  t.batch_size, t.learning_rate, t.train_iteration = 16, 1e-3, 30
  seqs, ids = synth_training_set(7000, 12, n_frames=40, dim=512, n_spk=3, mean_run=6, noise=0.02)
  model.fit(seqs, ids, t)
  om = uis_oracle.OracleModel(model.export_weights())
  x = synth_utt(7200, n_frames=40, dim=512, n_spk=4, mean_run=6, noise=0.02)[0]
  i.beam_size, i.look_ahead, i.test_iteration = 10, 3, 1
  monkeypatch.setenv('UISRNN_B200_TREE_SPILL', '0')
  with pytest.raises(RuntimeError):
    model.predict(x, i)
  monkeypatch.delenv('UISRNN_B200_TREE_SPILL')
  want = uis_oracle.predict_single(om, x, beam_size=10, look_ahead=3, test_iteration=1)
  assert len(set(want)) >= 3
  assert model.predict(x, i) == want


# ---- 6. budget exhaustion ---------------------------------------------------------------------------------------

def test_exhausted_arena_budget_fails_loudly_then_recovers(native, monkeypatch):
  _, model, om = _cached(native, 1024, 512, 2)
  xs = utterances(512, 720, (30,))
  monkeypatch.setenv('UISRNN_B200_TREE_SPILL_MB', '1')
  with pytest.raises(native.NativeError) as ei:
    model.predict(xs, beam_size=10, look_ahead=3, test_iteration=1)
  assert ei.value.code == native.UIS_ERR_CAPACITY
  assert 'UISRNN_B200_TREE_SPILL_MB' in str(ei.value) and 'arena' in str(ei.value)
  monkeypatch.delenv('UISRNN_B200_TREE_SPILL_MB')
  got = model.predict(xs, beam_size=10, look_ahead=3, test_iteration=1)[0]
  assert got.tolist() == uis_oracle.predict_single(om, xs[0], beam_size=10, look_ahead=3, test_iteration=1)
