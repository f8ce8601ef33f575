"""Stacked GRUs (rnn_depth 2..4) and look-ahead trees (look_ahead >= 2) at the largest kernel shape, hidden 1024 /
dim 512, natively and zero-padded (512-d x-vectors at the default hidden size, hidden 600 / dim 300).  Every decode
is compared with the CPU oracle at the model's ORIGINAL shape: labels identical, per-step scores within 1e-5
relative, the best hypothesis's hidden states (every layer) and running means within 1e-5 absolute.

The synthetic models are untrained; sigma2 = 0.003 and transition_bias 0.3 keep their decodes non-trivial (several
clusters, several distinct labels in the returned slice), which every case checks so that none passes vacuously."""
import random

import numpy as np
import pytest

from helpers import compare_trace, rel_err, uis_oracle

pytestmark = pytest.mark.gpu

SCORE_RTOL = 1e-5
STATE_ATOL = 1e-5


@pytest.fixture(scope='module')
def native():
  from uisrnn_b200 import native as nat
  nat.load_library()
  return nat


def large_model(H, D, depth, seed, sigma2=0.003, transition_bias=0.3):
  rng = np.random.default_rng(seed)
  u = lambda *s: (rng.uniform(-1, 1, size=s) / np.sqrt(H)).astype(np.float32)
  w = {'depth': depth, 'w1': u(H, H), 'b1': u(H), 'w2': u(D, H), 'b2': u(D), 'h0': u(depth, 1, H),
       'sigma2': np.full(D, sigma2, np.float32), 'transition_bias': transition_bias, 'crp_alpha': 1.0}
  for l in range(depth):
    w['weight_ih_l%d' % l] = u(3 * H, D if l == 0 else H)
    w['weight_hh_l%d' % l] = u(3 * H, H)
    w['bias_ih_l%d' % l] = u(3 * H)
    w['bias_hh_l%d' % l] = u(3 * H)
  return w


def utterances(D, seed, lengths):
  """Unit-norm frames around unit-norm speaker centres, speaker runs of about 6 frames."""
  from uisrnn_b200.synth import synth_utt
  return [synth_utt(seed + i, n_frames=n, dim=D, n_spk=4, mean_run=6, noise=0.02)[0] for i, n in enumerate(lengths)]


_MODELS = {}


def _cached(native, H, D, depth):
  key = (H, D, depth)
  if key not in _MODELS:
    w = large_model(H, D, depth, seed=H + D + depth)
    _MODELS[key] = (w, native.NativeModel(w), uis_oracle.OracleModel(w))
  return _MODELS[key]


def check_against_oracle(native, H, D, depth, beam, la, titer, lengths, seed, kcap=None, min_distinct=3):
  """Decodes `lengths` fresh utterances (the first one traced) and checks them against the oracle.  kcap defaults to
  64 at look_ahead 1 (room for every cluster these decodes open) and to the library's 16 for the tree kernel (whose
  node capacity shrinks as the tables grow)."""
  if kcap is None:
    kcap = 64 if la == 1 else 0
  w, model, om = _cached(native, H, D, depth)
  xs = utterances(D, seed, lengths)
  got, dbg = model.predict(xs, beam_size=beam, look_ahead=la, test_iteration=titer, kcap=kcap, trace_utt=0)
  assert model.stats()['engine'] == 1
  for i, (x, g) in enumerate(zip(xs, got)):
    rec = {} if i == 0 else None
    want = uis_oracle.predict_single(om, x, beam_size=beam, look_ahead=la, test_iteration=titer, record=rec)
    assert g.tolist() == want, 'utterance %d' % i
    if i == 0:
      assert len(set(want)) >= min_distinct, 'trivial decode: %s' % want
      compare_trace(dbg['win'], dbg['score'], dbg['off'], rec['win'], rec['score'], rec['off'], rtol=SCORE_RTOL)
      nb = len(rec['final_scores'])
      assert rel_err(dbg['final_scores'][0][:nb], rec['final_scores']) < SCORE_RTOL
      assert dbg['best_hidden'].shape == rec['final_hidden'].shape == (len(rec['final_mean']), depth, H)
      assert dbg['best_mean'].shape == rec['final_mean'].shape
      assert np.max(np.abs(dbg['best_hidden'] - rec['final_hidden'])) < STATE_ATOL
      assert np.max(np.abs(dbg['best_mean'] - rec['final_mean'])) < STATE_ATOL
      assert np.array_equal(dbg['best_blocks'], rec['final_blocks'])
  return model


@pytest.mark.parametrize('depth,seed', [(2, 120), (3, 135), (4, 140)])
@pytest.mark.parametrize('beam,titer', [(5, 1), (5, 2), (10, 1), (10, 2)])
def test_stacked_layers_at_1024x512(native, depth, seed, beam, titer):
  """The inputs are seeded so that no two hypotheses tie at the beam cut-off within fp32 rounding: GPU and oracle sum
  the GRU products in different orders (scores agree to ~2e-7 relative), so such a tie may keep either hypothesis."""
  check_against_oracle(native, 1024, 512, depth, beam, 1, titer, (40, 17), seed=seed)


@pytest.mark.parametrize('depth,la,beam', [(1, 2, 10), (1, 3, 3), (2, 2, 10), (2, 3, 3), (1, 2, 30)])
def test_look_ahead_at_1024x512(native, depth, la, beam):
  """The look-ahead tree kernel at 8 columns per weight pass; beam 30 / look_ahead 2 is the shape of BASELINE config 3.
  At look_ahead 3 a step's tree holds about beam * K^2 nodes (K clusters per hypothesis), so beam 3 on 12 frames keeps
  it within the on-chip node arrays (about 350 nodes at this shape)."""
  check_against_oracle(native, 1024, 512, depth, beam, la, 1, (24, 7) if la == 2 else (12, 7), seed=200 + 10 * depth + la)


@pytest.mark.parametrize('H,D,depth,la', [(512, 512, 3, 1), (600, 300, 2, 2)])
def test_padded_models_run_in_the_1024x512_kernels(native, H, D, depth, la):
  """512-d embeddings at the default hidden size (the x-vector case) and an odd shape, zero-padded to (1024, 512):
  the un-padded states of every layer come back through the taps."""
  check_against_oracle(native, H, D, depth, 10, la, 2 if la == 1 else 1, (40 if la == 1 else 30, 9), seed=300 + H)


def test_wide_beam_on_a_deep_model(native):
  """beam 64 at depth 2: the per-hypothesis tables of 64 hypotheses do not fit shared memory at the default kcap, so
  the library shrinks kcap itself.  16 frames at test_iteration 1 cannot open more clusters than that."""
  check_against_oracle(native, 1024, 512, 2, 64, 1, 1, (16, 5), seed=400, kcap=0)


def test_batching_independence_at_depth_2(native):
  w, model, _ = _cached(native, 1024, 512, 2)
  xs = utterances(512, 500, (23, 0, 1, 40, 9, 31, 2, 18))
  together = model.predict(xs, beam_size=10, test_iteration=2)
  assert len(together[1]) == 0 and len(together[2]) == 1
  assert len(set(together[3].tolist())) >= 3
  few_ctas = model.predict(xs, beam_size=10, test_iteration=2, n_ctas=3)
  for got in [few_ctas] + [model.predict(xs, beam_size=10, test_iteration=2, n_ctas=3, lanes=g) for g in (1, 2)]:
    assert all(a.tolist() == b.tolist() for a, b in zip(got, together))
  for i in range(len(xs)):
    assert model.predict([xs[i]], beam_size=10, test_iteration=2)[0].tolist() == together[i].tolist()


def test_errors_still_fail_loudly(native, monkeypatch):
  from helpers import inference_args, uisrnn_from_weights
  from uisrnn_b200 import uisrnn as impl
  w, model, om = _cached(native, 1024, 512, 2)
  x = utterances(512, 600, (40,))[0]
  for la in (1, 2):
    with pytest.raises(native.NativeError) as ei:
      model.predict([x], beam_size=10, look_ahead=la, test_iteration=1, kcap=1)
    assert ei.value.code == native.UIS_ERR_OVERFLOW
  # the public API grows kcap and retries: start it at 1 so that the first attempt overflows
  monkeypatch.setattr(impl, '_DEFAULT_KCAP', 1)
  api = uisrnn_from_weights(w, enable_cuda=True)
  for la in (1, 2):
    want = uis_oracle.predict_single(om, x, beam_size=10, look_ahead=la, test_iteration=1)
    assert len(set(want)) >= 3
    assert api.predict(x, inference_args(10, la, 1)) == want
  with pytest.raises(native.NativeError) as ei:
    native.NativeModel(large_model(1100, 512, 2, seed=1))
  assert ei.value.code == native.UIS_ERR_UNSUPPORTED


def test_fit_then_predict_512d_depth2_through_the_api(capsys):
  """The x-vector case end to end on CUDA: construction logs no warning, fit() trains on the device, and predict()
  (look_ahead 1 and 2) equals the oracle on the trained weights."""
  import torch
  import uisrnn
  from uisrnn_b200.synth import synth_training_set, synth_utt
  np.random.seed(7); random.seed(7); torch.manual_seed(7)
  m, t, i = uisrnn.parse_arguments([])
  m.observation_dim, m.rnn_hidden_size, m.rnn_depth, m.verbosity = 512, 512, 2, 3
  m.sigma2 = 0.003
  capsys.readouterr()
  model = uisrnn.UISRNN(m)
  assert model.device.type == 'cuda'
  assert 'Warning' not in capsys.readouterr().out
  model.logger.verbosity = 0
  t.batch_size, t.learning_rate, t.train_iteration = 16, 1e-3, 30
  seqs, ids = synth_training_set(7000, 12, n_frames=40, dim=512, n_spk=3, mean_run=6, noise=0.02)
  model.fit(seqs, ids, t)
  assert model.last_fit_backend == 'native'
  om = uis_oracle.OracleModel(model.export_weights())
  x = synth_utt(7100, n_frames=30, dim=512, n_spk=4, mean_run=6, noise=0.02)[0]
  for la in (1, 2):
    i.beam_size, i.look_ahead, i.test_iteration = 10, la, 1
    want = uis_oracle.predict_single(om, x, beam_size=10, look_ahead=la, test_iteration=1)
    assert model.predict(x, i) == want
    assert model.predict([x, x[:5]], i)[0] == want
