"""GPU parity tests: the sm_90a path, called through the C ABI (ctypes -> libuisrnn_b200.so),
against (a) golden vectors produced by the unmodified reference and (b) the CPU oracle on fresh
seeded inputs.  Labels must be identical; scores within 1e-5 relative; GRU hidden states and
running means within 1e-5 absolute (BASELINE.md section 3.4)."""
import numpy as np
import pytest

import beam_replay
from helpers import (GOLDEN, compare_trace, depth2_cases, load_weights, oracle_model, rel_err, small_cases,
                     toy_utterances, uis_oracle)

pytestmark = pytest.mark.gpu

SCORE_RTOL = 1e-5
STATE_ATOL = 1e-5


@pytest.fixture(scope='module')
def native():
  from uisrnn_b200 import native as nat
  nat.load_library()
  return nat


@pytest.fixture(scope='module')
def small_model(native):
  return native.NativeModel(load_weights('model_small.npz'))


@pytest.fixture(scope='module')
def toy_model(native):
  return native.NativeModel(load_weights('model_toy100.npz'))


def test_model_constants_match_oracle(small_model, toy_model):
  for nm, name in ((small_model, 'model_small.npz'), (toy_model, 'model_toy100.npz')):
    om = oracle_model(name)
    mean0, hidden0 = nm.constants()
    assert np.max(np.abs(mean0 - om.mean0)) < STATE_ATOL
    assert np.max(np.abs(hidden0 - om.hidden0)) < STATE_ATOL


@pytest.mark.parametrize('case', small_cases(), ids=lambda c: c['name'])
def test_small_cases_match_reference_golden(small_model, case):
  """Beam sizes 1/3/10/30, look_ahead 1/2/3 (incl. a shorter tail chunk), test_iteration 1/2/3."""
  labs, dbg = small_model.predict([case['x']], beam_size=case['beam_size'], look_ahead=case['look_ahead'],
                                  test_iteration=case['test_iteration'], trace_utt=0)
  assert labs[0].tolist() == case['labels'].tolist()
  swaps = compare_trace(dbg['win'], dbg['score'], dbg['off'], case['win'], case['score'], case['off'],
                        rtol=SCORE_RTOL)
  if case['beam_size'] <= 10:
    assert swaps == 0  # no near-ties in these fixtures: winners identical, in order
  nb = len(case['final_scores'])
  assert rel_err(dbg['final_scores'][0][:nb], case['final_scores']) < SCORE_RTOL
  assert np.all(np.isinf(dbg['final_scores'][0][nb:]))
  assert np.max(np.abs(dbg['best_hidden'] - case['final_hidden'])) < STATE_ATOL
  assert np.max(np.abs(dbg['best_mean'] - case['final_mean'])) < STATE_ATOL
  assert np.array_equal(dbg['best_blocks'], case['final_blocks'])


def test_toy_testing_data_labels_identical_to_reference(toy_model):
  """North star: integer-exact labels on all 25 utterances of data/toy_testing_data.npz."""
  xs, labs = toy_utterances()
  got = toy_model.predict(xs)
  for i, (g, want) in enumerate(zip(got, labs)):
    assert g.tolist() == want.tolist(), 'utterance %d' % i
  st = toy_model.stats()
  assert st['frames'] == sum(len(x) for x in xs) and st['beam_steps'] == 2 * st['frames']


@pytest.mark.parametrize('idx', [0, 1])
def test_toy_trace_matches_reference(toy_model, idx):
  xs, _ = toy_utterances()
  g = np.load(GOLDEN + '/toy_trace.npz')
  _, dbg = toy_model.predict([xs[idx]], trace_utt=0)
  compare_trace(dbg['win'], dbg['score'], dbg['off'], g['u%d_win' % idx], g['u%d_score' % idx],
                g['u%d_off' % idx], rtol=SCORE_RTOL)
  assert np.max(np.abs(dbg['best_hidden'] - g['u%d_final_hidden' % idx])) < STATE_ATOL
  assert np.max(np.abs(dbg['best_mean'] - g['u%d_final_mean' % idx])) < STATE_ATOL


def test_synth500_labels_identical_to_reference(toy_model):
  """BASELINE config 2 shape (500-frame, 256-d, beam 10): reference labels are golden."""
  from uisrnn_b200.synth import synth_utt
  g = np.load(GOLDEN + '/synth500.npz')
  xs = [synth_utt(int(s))[0] for s in g['seeds']]
  got = toy_model.predict(xs)
  for o, want in zip(got, g['labels']):
    assert o.tolist() == want.tolist()


@pytest.mark.parametrize('beam,titer', [(10, 2), (4, 1), (32, 2), (1, 2)])
def test_fresh_inputs_match_oracle(small_model, beam, titer):
  from uisrnn_b200.synth import synth_utt
  om = oracle_model('model_small.npz')
  xs = [synth_utt(9000 + i, n_frames=n, dim=64, n_spk=k, noise=0.08)[0]
        for i, (n, k) in enumerate([(70, 3), (1, 1), (33, 2), (120, 4), (2, 2), (64, 3)])]
  got = small_model.predict(xs, beam_size=beam, test_iteration=titer)
  for x, o in zip(xs, got):
    want = uis_oracle.predict_single(om, x, beam_size=beam, look_ahead=1, test_iteration=titer)
    assert o.tolist() == want


def test_ragged_and_empty_batch(small_model):
  from uisrnn_b200.synth import synth_utt
  assert small_model.predict([]) == []
  xs = [np.zeros((0, 64)), synth_utt(1, n_frames=5, dim=64)[0]]
  got = small_model.predict(xs)
  assert len(got[0]) == 0 and len(got[1]) == 5


def test_many_utterances_are_independent_of_batching(toy_model):
  """Size-independent property: predict(list) == [predict(x) for x in list], any CTA count."""
  from uisrnn_b200.synth import synth_utt
  xs = [synth_utt(3000 + i, n_frames=40 + 7 * (i % 5))[0] for i in range(40)]
  together = toy_model.predict(xs)
  few_ctas = toy_model.predict(xs, n_ctas=3)
  for lanes in (1, 2, 3):  # lanes share weight passes only; results must not depend on them
    got = toy_model.predict(xs, n_ctas=5, lanes=lanes, engine=1)
    assert toy_model.stats()["lanes"] == min(lanes, 2)  # SMEM limits lanes to 2 at kcap=32
    assert all(a.tolist() == b.tolist() for a, b in zip(got, together)), 'lanes=%d' % lanes
  for i in (0, 7, 39):
    alone = toy_model.predict([xs[i]])[0]
    assert alone.tolist() == together[i].tolist() == few_ctas[i].tolist()
  # permutation invariance of the result
  perm = np.random.default_rng(0).permutation(len(xs))
  shuffled = toy_model.predict([xs[i] for i in perm])
  for j, i in enumerate(perm):
    assert shuffled[j].tolist() == together[i].tolist()


def test_kcap_overflow_fails_loudly(small_model, native):
  from uisrnn_b200.synth import synth_utt
  x = synth_utt(77, n_frames=60, dim=64, n_spk=4, noise=0.08)[0]
  with pytest.raises(native.NativeError) as ei:
    small_model.predict([x], kcap=1)
  assert ei.value.code == native.UIS_ERR_OVERFLOW


def test_unsupported_options_fail_loudly(small_model, native):
  x = np.zeros((4, 64))
  with pytest.raises(native.NativeError) as ei:
    small_model.predict([x], look_ahead=9)
  assert ei.value.code == native.UIS_ERR_UNSUPPORTED
  with pytest.raises(native.NativeError) as ei:
    small_model.predict([x], beam_size=129)                  # look_ahead 1 serves beam_size <= 128
  assert ei.value.code == native.UIS_ERR_UNSUPPORTED
  with pytest.raises(native.NativeError) as ei:
    small_model.predict([x], beam_size=33, look_ahead=2)     # the look-ahead tree kernel: beam_size <= 32
  assert ei.value.code == native.UIS_ERR_UNSUPPORTED
  with pytest.raises(native.NativeError):
    small_model.predict([x], beam_size=0)


@pytest.mark.parametrize('beam,la,titer', [(10, 2, 2), (6, 3, 1), (30, 2, 1), (3, 4, 1)])
def test_look_ahead_fresh_inputs_match_oracle(small_model, beam, la, titer):
  from uisrnn_b200.synth import synth_utt
  om = oracle_model('model_small.npz')
  xs = [synth_utt(9500 + i, n_frames=n, dim=64, n_spk=k, noise=0.08)[0]
        for i, (n, k) in enumerate([(31, 3), (1, 1), (24, 2), (3, 2)])]
  got = small_model.predict(xs, beam_size=beam, look_ahead=la, test_iteration=titer)
  for x, o in zip(xs, got):
    want = uis_oracle.predict_single(om, x, beam_size=beam, look_ahead=la, test_iteration=titer)
    assert o.tolist() == want


@pytest.mark.parametrize('beam,engine', [(33, 1), (40, 0), (64, 1), (100, 1), (128, 0)])
def test_beams_wider_than_32_match_oracle(small_model, beam, engine):
  """beam_size > 32 (any int in the reference, arguments.py:175-180): phase P3 walks the winners in chunks of 32 and
  the candidate records carry a 7-bit hypothesis index.  Labels against the oracle; a hand-picked kcap keeps the
  per-hypothesis tables (B * kcap entries) inside shared memory."""
  from uisrnn_b200.synth import synth_utt
  om = oracle_model('model_small.npz')
  xs = [synth_utt(9700 + i, n_frames=n, dim=64, n_spk=k, noise=0.08)[0]
        for i, (n, k) in enumerate([(40, 3), (1, 1), (23, 2), (57, 4)])]
  got = small_model.predict(xs, beam_size=beam, look_ahead=1, test_iteration=2, engine=engine)
  st = small_model.stats()
  assert st['engine'] == (engine or st['engine'])
  for x, o in zip(xs, got):
    assert o.tolist() == uis_oracle.predict_single(om, x, beam_size=beam, look_ahead=1, test_iteration=2)


@pytest.mark.parametrize('engine', [1, 2])
def test_beam_64_default_shape_matches_oracle(toy_model, engine):
  """Both engines at the default shape; on the tensor-core engine a lane's columns (up to 65) span two passes."""
  from uisrnn_b200.synth import synth_utt
  om = oracle_model('model_toy100.npz')
  xs = [synth_utt(4321 + i, n_frames=30)[0] for i in range(3)]
  got = toy_model.predict(xs, beam_size=64, look_ahead=1, test_iteration=2, engine=engine)
  assert toy_model.stats()['engine'] == engine
  for x, o in zip(xs, got):
    assert o.tolist() == uis_oracle.predict_single(om, x, beam_size=64, look_ahead=1, test_iteration=2)


def test_wide_beam_look_ahead_config3_shape(toy_model):
  """BASELINE config 3 (beam_size=30, look_ahead=2, hidden=512) on a short utterance vs the oracle."""
  from uisrnn_b200.synth import synth_utt
  om = oracle_model('model_toy100.npz')
  x = synth_utt(1234, n_frames=24)[0]
  got = toy_model.predict([x], beam_size=30, look_ahead=2, test_iteration=2)[0]
  assert got.tolist() == uis_oracle.predict_single(om, x, beam_size=30, look_ahead=2, test_iteration=2)


def _random_weights(H, D, seed, scale=1.0):
  """A synthetic (untrained) model: small recurrent weights so hidden states stay informative."""
  rng = np.random.default_rng(seed)
  u = lambda *s: (rng.uniform(-1, 1, size=s) * scale / np.sqrt(H)).astype(np.float32)
  return {'depth': 1, 'weight_ih_l0': u(3 * H, D), 'weight_hh_l0': u(3 * H, H), 'bias_ih_l0': u(3 * H),
          'bias_hh_l0': u(3 * H), 'w1': u(H, H), 'b1': u(H), 'w2': u(D, H), 'b2': u(D),
          'h0': u(1, 1, H), 'sigma2': (0.05 + 0.1 * rng.random(D)).astype(np.float32),
          'transition_bias': 0.2, 'crp_alpha': 0.7}


def test_models_above_the_default_shape_run_in_the_1024x512_kernel(native):
  """hidden up to 1024 / dim up to 512 (arguments.py:44-54 takes any int): the (1024, 512) instantiation of the fp32
  FFMA engine, natively and zero-padded (hidden 600 / dim 300), against the oracle; above that the library refuses."""
  rng = np.random.default_rng(11)
  for H, D in ((1024, 512), (600, 300)):
    w = _random_weights(H, D, seed=H + D)
    model = native.NativeModel(w)
    om = uis_oracle.OracleModel(w)
    xs = [rng.standard_normal((n, D)) * 0.3 for n in (9, 4)]
    got = model.predict(xs, beam_size=5, look_ahead=1, test_iteration=2, kcap=64)
    assert model.stats()['engine'] == 1
    for x, o in zip(xs, got):
      assert o.tolist() == uis_oracle.predict_single(om, x, beam_size=5, look_ahead=1, test_iteration=2)
  with pytest.raises(native.NativeError) as ei:
    native.NativeModel(_random_weights(1100, 256, seed=1))
  assert ei.value.code == native.UIS_ERR_UNSUPPORTED


@pytest.mark.parametrize('H,D', [(256, 128), (128, 64), (512, 256)])
def test_random_models_all_kernel_shapes_match_oracle(native, H, D):
  """Every instantiated (hidden, dim) pair, untrained weights (cluster counts grow quickly here, so
  the table-overflow path and many-cluster scoring are exercised), crp_alpha != 1."""
  w = _random_weights(H, D, seed=H + D)
  model = native.NativeModel(w)
  om = uis_oracle.OracleModel(w)
  rng = np.random.default_rng(7)
  xs = [rng.standard_normal((n, D)) * 0.3 for n in (17, 5, 26)]
  for beam, la in ((10, 1), (4, 2)):
    try:
      got = model.predict(xs, beam_size=beam, look_ahead=la, test_iteration=2, kcap=64 if la == 1 else 48)
    except native.NativeError as err:  # a legitimately huge tree is reported, never mis-computed
      assert err.code in (native.UIS_ERR_CAPACITY, native.UIS_ERR_OVERFLOW)
      continue
    for x, o in zip(xs, got):
      assert o.tolist() == uis_oracle.predict_single(om, x, beam_size=beam, look_ahead=la, test_iteration=2)


def test_test_iteration_is_tiling_full_size(toy_model):
  """Full-size property check (no oracle): test_iteration=2 must equal decoding the utterance
  concatenated with itself at test_iteration=1 and keeping the labels of the last copy
  (uisrnn.py:524, :561)."""
  from uisrnn_b200.synth import synth_utt
  x = synth_utt(4321, n_frames=700)[0]
  twice = toy_model.predict([np.concatenate([x, x])], test_iteration=1)[0]
  tiled = toy_model.predict([x], test_iteration=2)[0]
  assert tiled.tolist() == twice[700:].tolist()


@pytest.mark.parametrize('case', depth2_cases(), ids=lambda c: c['name'])
def test_depth2_matches_reference_golden(native, case):
  """Stacked GRU (rnn_depth=2): labels, per-step winners and both layers' hidden states against the
  unmodified reference (look_ahead 1 and 2)."""
  model = native.NativeModel(load_weights('model_small_d2.npz'))
  labs, dbg = model.predict([case['x']], beam_size=case['beam_size'], look_ahead=case['look_ahead'],
                            test_iteration=case['test_iteration'], trace_utt=0)
  assert labs[0].tolist() == case['labels'].tolist()
  compare_trace(dbg['win'], dbg['score'], dbg['off'], case['win'], case['score'], case['off'], rtol=SCORE_RTOL)
  assert dbg['best_hidden'].shape == case['final_hidden'].shape
  assert np.max(np.abs(dbg['best_hidden'] - case['final_hidden'])) < STATE_ATOL
  assert np.max(np.abs(dbg['best_mean'] - case['final_mean'])) < STATE_ATOL


def test_depth3_untrained_matches_oracle(native):
  rng = np.random.default_rng(3)
  H, D, depth = 128, 64, 3
  u = lambda *s: (rng.uniform(-1, 1, size=s) / np.sqrt(H)).astype(np.float32)
  w = {'depth': depth, 'w1': u(H, H), 'b1': u(H), 'w2': u(D, H), 'b2': u(D), 'h0': u(depth, 1, H),
       'sigma2': (0.05 + 0.1 * rng.random(D)).astype(np.float32), 'transition_bias': 0.15, 'crp_alpha': 1.0}
  for l in range(depth):
    w['weight_ih_l%d' % l] = u(3 * H, D if l == 0 else H); w['weight_hh_l%d' % l] = u(3 * H, H)
    w['bias_ih_l%d' % l] = u(3 * H); w['bias_hh_l%d' % l] = u(3 * H)
  model = native.NativeModel(w)
  om = uis_oracle.OracleModel(w)
  x = rng.standard_normal((21, D)) * 0.3
  got = model.predict([x], beam_size=6, test_iteration=2, kcap=64)[0]
  assert got.tolist() == uis_oracle.predict_single(om, x, beam_size=6, look_ahead=1, test_iteration=2)


@pytest.mark.parametrize('H,D,depth', [(100, 40, 1), (8, 2, 2), (300, 200, 1), (129, 65, 1), (512, 100, 1), (24, 16, 3)])
def test_any_shape_up_to_512x256_runs_zero_padded(native, H, D, depth):
  """A model whose (hidden, dim) is not a kernel shape runs zero-padded in the next larger one (uis_model_create):
  labels against the oracle at the ORIGINAL shape, and the traced utterance's per-step scores and selection and the
  un-padded states of its best hypothesis against the float64 replay (tests/beam_replay.py) at that shape.
  (8, 2, depth 2) is the model of the reference's own integration test; observation_dim 16 / 100 are its other shapes."""
  rng = np.random.default_rng(1000 * H + D)
  u = lambda *s: (rng.uniform(-1, 1, size=s) / np.sqrt(H)).astype(np.float32)
  w = {'depth': depth, 'w1': u(H, H), 'b1': u(H), 'w2': u(D, H), 'b2': u(D), 'h0': u(depth, 1, H),
       'sigma2': (0.05 + 0.1 * rng.random(D)).astype(np.float32), 'transition_bias': 0.15, 'crp_alpha': 1.0}
  for l in range(depth):
    w['weight_ih_l%d' % l] = u(3 * H, D if l == 0 else H); w['weight_hh_l%d' % l] = u(3 * H, H)
    w['bias_ih_l%d' % l] = u(3 * H); w['bias_hh_l%d' % l] = u(3 * H)
  model = native.NativeModel(w)
  om = uis_oracle.OracleModel(w)
  mean0, hidden0 = model.constants()
  assert mean0.shape == (D,) and hidden0.shape == (depth, H)
  assert np.max(np.abs(mean0 - om.mean0)) < STATE_ATOL and np.max(np.abs(hidden0 - om.hidden0)) < STATE_ATOL
  centres = rng.standard_normal((3, D))
  xs = []
  for n in (31, 1, 18):
    lab = (np.arange(n) // 7) % 3
    xs.append(centres[lab] * 0.3 + 0.05 * rng.standard_normal((n, D)))
  got, dbg = model.predict(xs, beam_size=5, test_iteration=2, kcap=64, trace_utt=0)
  for x, o in zip(xs, got):
    assert o.tolist() == uis_oracle.predict_single(om, x, beam_size=5, look_ahead=1, test_iteration=2)
  assert dbg['best_mean'].shape[1] == D and dbg['best_hidden'].shape[1:] == (depth, H)
  # the taps: every step's increments and selection and the final state against the float64 replay at this shape
  final = dict(best_mean=dbg['best_mean'], best_hidden=dbg['best_hidden'], best_blocks=dbg['best_blocks'],
               final_k=dbg['final_k'][0], final_scores=dbg['final_scores'][0])
  replay = beam_replay.Replay(w, xs[0], 5, 1, 2, dbg['win'], dbg['score'], dbg['off'], mean0=mean0)
  beam_replay.check(replay, beam_replay.INC_RTOL, labels=got[0].tolist(), final=final,
                    state_tol=beam_replay.STATE_TOL)
  la2 = model.predict(xs[:1], beam_size=3, look_ahead=2, test_iteration=1, kcap=32)[0]
  assert la2.tolist() == uis_oracle.predict_single(om, xs[0], beam_size=3, look_ahead=2, test_iteration=1)


def test_shapes_beyond_the_largest_kernel_fail_loudly(native):
  H, D = 1152, 256
  z = lambda *s: np.zeros(s, np.float32)
  w = {'depth': 1, 'weight_ih_l0': z(3 * H, D), 'weight_hh_l0': z(3 * H, H), 'bias_ih_l0': z(3 * H), 'bias_hh_l0': z(3 * H),
       'w1': z(H, H), 'b1': z(H), 'w2': z(D, H), 'b2': z(D), 'h0': z(1, 1, H), 'sigma2': np.ones(D, np.float32),
       'transition_bias': 0.1, 'crp_alpha': 1.0}
  with pytest.raises(native.NativeError) as ei:
    native.NativeModel(w)
  assert ei.value.code == native.UIS_ERR_UNSUPPORTED
