"""The tensor-core engine of the look_ahead-1 beam kernel (`engine=2`: wgmma MMAs over fp16 hi/lo split operands,
register accumulators, tensor-map TMA -- uisrnn_b200/csrc/uis_beam_tc.cuh) against the same pins as the FFMA kernels:
labels produced by the unmodified reference (toy test set, 500-frame utterances of bench.py's workload), per-step
winners / scores / final hidden states of the reference's own trace (scores 1e-5 relative, states 1e-5 absolute,
BASELINE.md section 3.4), and the CPU oracle on the other tileable shape (256, 128)."""
import numpy as np
import pytest

from helpers import GOLDEN, compare_trace, load_weights, toy_utterances, uis_oracle

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


def _bench_golden():
  from uisrnn_b200.synth import synth_utt
  g = np.load(GOLDEN + '/synth500_bench.npz')
  xs = [synth_utt(int(s))[0] for s in g['seeds']]
  return [int(s) for s in g['seeds']], xs, [lab.tolist() for lab in g['labels']]


def test_toy_testing_data_labels_identical_to_reference(toy_model):
  xs, labs = toy_utterances()
  got = toy_model.predict(xs, engine=2)
  st = toy_model.stats()
  assert st['engine'] == 2 and st['tc_columns'] == 48 and st['cluster'] == 1
  for i, (g, want) in enumerate(zip(got, labs)):
    assert g.tolist() == want.tolist(), 'utterance %d' % i
  assert st['frames'] == sum(len(x) for x in xs) and st['beam_steps'] == 2 * st['frames']


@pytest.mark.parametrize('idx', [0, 1])
def test_toy_trace_matches_reference(toy_model, idx):
  """Per-step winners and scores of the reference's own trace; hidden states / means of the best hypothesis."""
  xs, _ = toy_utterances()
  g = np.load(GOLDEN + '/toy_trace.npz')
  _, dbg = toy_model.predict([xs[idx]], trace_utt=0, engine=2)
  assert toy_model.stats()['engine'] == 2
  compare_trace(dbg['win'], dbg['score'], dbg['off'], g['u%d_win' % idx], g['u%d_score' % idx],
                g['u%d_off' % idx], rtol=SCORE_RTOL)
  assert np.max(np.abs(dbg['best_hidden'] - g['u%d_final_hidden' % idx])) < STATE_ATOL
  assert np.max(np.abs(dbg['best_mean'] - g['u%d_final_mean' % idx])) < STATE_ATOL


@pytest.mark.parametrize('lanes,n_ctas', [(0, 0), (6, 2), (2, 0), (8, 1), (4, 3), (1, 0)])
def test_default_shape_500_frames_reference_labels(toy_model, lanes, n_ctas):
  """(512, 256), 1000 beam steps per utterance, lanes sharing one pass (incl. more columns than one pass holds)."""
  from uisrnn_b200.synth import synth_utt
  _, xs, want = _bench_golden()
  g2 = np.load(GOLDEN + '/synth500.npz')
  xs = xs + [synth_utt(int(s))[0] for s in g2['seeds']]
  want = want + [lab.tolist() for lab in g2['labels']]
  got = toy_model.predict(xs, engine=2, lanes=lanes, n_ctas=n_ctas)
  st = toy_model.stats()
  assert st['engine'] == 2 and st['tc_columns'] == 48
  if lanes:
    assert st['lanes'] <= lanes
  for i, (g, w) in enumerate(zip(got, want)):
    assert g.tolist() == w, 'utterance %d' % i


def test_engines_agree_on_a_ragged_batch(toy_model):
  """Size-independent property: the FFMA and the tensor-core engine give the same labels on every utterance of a
  ragged batch (empty and one-frame utterances included), whatever the lane count."""
  from uisrnn_b200.synth import synth_utt
  xs = [synth_utt(3000 + i, n_frames=[40, 1, 75, 0, 12, 131, 64, 2][i % 8])[0] if [40, 1, 75, 0, 12, 131, 64, 2][i % 8]
        else np.zeros((0, 256)) for i in range(48)]
  ffma = toy_model.predict(xs, engine=1)
  assert toy_model.stats()['engine'] == 1
  for lanes, n_ctas in ((0, 4), (3, 7), (6, 0)):
    tc = toy_model.predict(xs, engine=2, lanes=lanes, n_ctas=n_ctas)
    assert toy_model.stats()['engine'] == 2
    assert all(a.tolist() == b.tolist() for a, b in zip(tc, ffma)), (lanes, n_ctas)


def _random_weights(H, D, seed):
  rng = np.random.default_rng(seed)
  u = lambda *s: (rng.uniform(-1, 1, size=s) / np.sqrt(H)).astype(np.float32)
  return {'depth': 1, 'weight_ih_l0': u(3 * H, D), 'weight_hh_l0': u(3 * H, H), 'bias_ih_l0': u(3 * H),
          'bias_hh_l0': u(3 * H), 'w1': u(H, H), 'b1': u(H), 'w2': u(D, H), 'b2': u(D),
          'h0': (3.0 * u(1, 1, H)), 'sigma2': (0.05 + 0.1 * rng.random(D)).astype(np.float32),
          'transition_bias': 0.1, 'crp_alpha': 1.0}


@pytest.mark.parametrize('H,D', [(256, 128), (512, 256)])
def test_untrained_models_match_oracle(native, H, D):
  """No reference-trained fixture for (256, 128): untrained weights (other scales, |h0| > 1 off the unit range the
  operand scale is derived from, many clusters) against the oracle; kcap given explicitly."""
  w = _random_weights(H, D, 11)
  model = native.NativeModel(w)
  om = uis_oracle.OracleModel(w)
  rng = np.random.default_rng(5)
  centres = rng.standard_normal((3, D))
  xs = []
  for n in (120, 97, 120, 64, 120, 33):
    lab = (np.arange(n) // 11) % 3
    xs.append(centres[lab] * 0.3 + 0.05 * rng.standard_normal((n, D)))
  got = model.predict(xs, kcap=64, engine=2, n_ctas=2)
  assert model.stats()['engine'] == 2
  for x, o in zip(xs, got):
    assert o.tolist() == uis_oracle.predict_single(om, x, beam_size=10, look_ahead=1, test_iteration=2)


def test_other_beam_sizes_match_oracle(toy_model):
  from uisrnn_b200.synth import synth_utt
  om = uis_oracle.OracleModel(load_weights('model_toy100.npz'))
  xs = [synth_utt(9100 + i, n_frames=60)[0] for i in range(4)]
  for beam, titer in ((1, 2), (4, 1), (32, 2)):
    got = toy_model.predict(xs, beam_size=beam, test_iteration=titer, engine=2, n_ctas=2)
    assert toy_model.stats()['engine'] == 2
    for x, o in zip(xs, got):
      assert o.tolist() == uis_oracle.predict_single(om, x, beam_size=beam, look_ahead=1, test_iteration=titer)


def test_table_overflow_and_unsupported_fail_loudly(toy_model, native):
  from uisrnn_b200.synth import synth_utt
  x = synth_utt(77, n_frames=60)[0]
  with pytest.raises(native.NativeError) as ei:
    toy_model.predict([x], kcap=1, engine=2)
  assert ei.value.code == native.UIS_ERR_OVERFLOW
  with pytest.raises(native.NativeError) as ei:
    toy_model.predict([x], look_ahead=2, engine=2)
  assert ei.value.code == native.UIS_ERR_UNSUPPORTED
  small = native.NativeModel(load_weights('model_small.npz'))  # (128, 64) does not tile by 128 rows
  with pytest.raises(native.NativeError) as ei:
    small.predict([np.zeros((4, 64))], engine=2)
  assert ei.value.code == native.UIS_ERR_UNSUPPORTED


def test_full_bench_batch_through_the_public_api(toy_model):
  """bench.py's per-GPU batch through uisrnn.UISRNN.predict (automatic engine = tensor cores): the utterances the
  reference decoded must come out identical; device-resident and host entry points agree on every utterance."""
  import torch
  from helpers import uisrnn_from_weights
  from uisrnn_b200.synth import synth_utt
  import uisrnn
  seeds, _, want = _bench_golden()
  U = 888
  xs = [synth_utt(100000 + u)[0] for u in range(U)]
  model = uisrnn_from_weights(load_weights('model_toy100.npz'), enable_cuda=True)
  _, _, iargs = uisrnn.parse_arguments([])
  got = model.predict(xs, iargs)
  st = model._native_model().stats()  # pylint: disable=protected-access
  assert st['engine'] == 2 and st['lanes'] == 6 and st['utterances'] == U
  for s, w in zip(seeds, want):
    assert got[s - 100000] == w, 'utterance %d of the bench batch' % (s - 100000)
  x_dev = torch.from_numpy(np.concatenate(xs).astype(np.float32)).cuda()
  lab_dev = torch.empty(U * 500, dtype=torch.int32, device='cuda')
  toy_model.predict_device(x_dev.data_ptr(), np.arange(U + 1, dtype=np.int64) * 500, lab_dev.data_ptr())
  assert toy_model.stats()['engine'] == 2
  assert np.array_equal(lab_dev.cpu().numpy(), np.concatenate([np.asarray(g, np.int32) for g in got]))
