"""Decoding-parameter sweeps without a GPU: the CPU decoder and scorer with crp_alpha / transition_bias overrides
against the numpy oracle and the float64 replay model built from a weights dict holding the pair, UISRNN.predict /
score(decode_params=...) against per-pair models, argument checking, and the sweep entry points of the C ABI."""
import ctypes
import os
import re
import warnings

import numpy as np
import pytest

import beam_replay
from helpers import GOLDEN, ROOT, inference_args, load_weights, toy_utterances, uis_oracle, uisrnn_from_weights

# the model's own pair first; the others are far enough apart that every pair's labels differ from every other's on
# at least one utterance (checked below), so a config mix-up cannot go unseen
PAIRS = [(1.0, 0.06358747231888642), (1e-3, 0.5), (30.0, 0.01), (0.2, 0.9)]


def utterances(n=3, frames=24):
  from uisrnn_b200.synth import synth_utt
  return [synth_utt(900 + i, n_frames=frames, dim=64, n_spk=3, noise=0.3)[0] for i in range(n)]


def with_pair(weights, pair):
  w = dict(weights)
  w['crp_alpha'], w['transition_bias'] = pair
  return w


@pytest.fixture(scope='module')
def small():
  return load_weights('model_small.npz')


def sweep_golden():
  """tests/golden/sweep_cases.npz (tools/make_sweep_golden.py): the reference's decodes and losses under non-default
  pairs.  Returns (toy, small, scores):
    toy    dict(pairs, utts, xs, labels[c][i]) -- predict_single labels of toy_test utterances utts[i] under pair c
    small  dict(pairs, xs, args, traces[c][i]) -- look_ahead-2 traces (labels, win, score, off, final_scores)
    scores list of dict(name, pair, model, x, labels, score, frames) -- per-frame losses of given labellings"""
  from uisrnn_b200.synth import synth_utt
  g = np.load(os.path.join(GOLDEN, 'sweep_cases.npz'))
  txs = toy_utterances()[0]
  utts = [int(u) for u in g['toy_utts']]
  lens = np.cumsum([0] + [len(txs[u]) for u in utts])
  toy = dict(pairs=[tuple(p) for p in g['toy_pairs']], utts=utts, xs=[txs[u] for u in utts],
             labels=[[row[lens[i]:lens[i + 1]] for i in range(len(utts))] for row in g['toy_labels']])
  off = np.cumsum(np.concatenate([[0], g['small_lengths']]))
  xs = [g['small_x'][off[i]:off[i + 1]].astype(np.float64) for i in range(len(off) - 1)]
  keys = ('labels', 'win', 'score', 'off', 'final_scores')
  small = dict(pairs=[tuple(p) for p in g['small_pairs']], xs=xs, args=[int(v) for v in g['small_args']],
               traces=[[{k: g['small_%d_%d_%s' % (c, i, k)] for k in keys} for i in range(len(xs))]
                       for c in range(len(g['small_pairs']))])
  scores = []
  for name in g['sc_names']:
    pre = 'sc_%s_' % name
    u = int(g[pre + 'toy_u'])
    if u >= 0:
      x = txs[u]
    else:
      seed, n, dim, n_spk, noise = g[pre + 'synth']
      x = synth_utt(int(seed), n_frames=int(n), dim=int(dim), n_spk=int(n_spk), noise=float(noise))[0]
      x = x.astype(np.float32).astype(np.float64)
    scores.append(dict(name=str(name), pair=tuple(g[pre + 'pair']), model=str(g[pre + 'model']), x=x,
                       labels=g[pre + 'labels'], score=float(g[pre + 'score']), frames=g[pre + 'frames']))
  return toy, small, scores


def test_fixture_own_pair_reproduces_toy_goldens():
  toy, small, _ = sweep_golden()
  g = np.load(os.path.join(GOLDEN, 'toy_test.npz'))
  off = np.concatenate([[0], np.cumsum(g['lengths'])])
  w = load_weights('model_toy100.npz')
  assert toy['pairs'][0] == (float(w['crp_alpha']), float(w['transition_bias']))
  for i, u in enumerate(toy['utts']):
    assert np.array_equal(toy['labels'][0][i], g['labels'][off[u]:off[u + 1]])
  for fixture in (toy['labels'], [[t['labels'] for t in row] for row in small['traces']]):
    for a in range(len(fixture)):
      for b in range(a):
        assert any(not np.array_equal(x, y) for x, y in zip(fixture[a], fixture[b])), (a, b)


def test_cpu_decoder_overrides_match_reference_traces(small):
  """The look_ahead-2 decodes of the D = 64 model under every pair: labels and final beam scores of the reference."""
  from uisrnn_b200 import beam_cpu
  _, fx, _ = sweep_golden()
  model = uisrnn_from_weights(small)
  b, la, ti = fx['args']
  for c, pair in enumerate(fx['pairs']):
    dec = beam_cpu.CpuBeamSearch(model, crp_alpha=pair[0], transition_bias=pair[1])
    for x, tr in zip(fx['xs'], fx['traces'][c]):
      labels, scores, _ = dec.decode(x, b, la, ti, n_best=b)
      assert labels[0] == tr['labels'].tolist(), pair
      want = tr['final_scores'][:len(scores)]
      assert np.allclose(scores, want, rtol=1e-5, atol=0), (pair, scores, want)


def test_cpu_score_overrides_match_reference_losses():
  """CpuBeamSearch.score with overrides gives the reference's per-frame losses bit for bit under non-default pairs
  (the 4400-frame case included: more than 4096 speaker turns)."""
  from uisrnn_b200 import beam_cpu
  _, _, cases = sweep_golden()
  for case in cases:
    model = uisrnn_from_weights(load_weights(case['model']))
    got, frames = beam_cpu.CpuBeamSearch(model, crp_alpha=case['pair'][0], transition_bias=case['pair'][1]).score(
        case['x'], case['labels'])
    assert np.array_equal(frames.view(np.uint32), case['frames'].view(np.uint32)), case['name']
    assert float(got) == case['score'], case['name']


def test_pairs_are_distinguishable(small):
  xs = utterances()
  labels = [[uis_oracle.predict_single(uis_oracle.OracleModel(with_pair(small, pr)), x, beam_size=5, look_ahead=1,
                                       test_iteration=2) for x in xs] for pr in PAIRS]
  for a in range(len(PAIRS)):
    for b in range(a + 1, len(PAIRS)):
      assert labels[a] != labels[b], (PAIRS[a], PAIRS[b])


@pytest.mark.parametrize('look_ahead', [1, 2])
def test_cpu_decoder_overrides_match_oracle(small, look_ahead):
  from uisrnn_b200 import beam_cpu
  model = uisrnn_from_weights(small)
  xs = utterances(2, 16 if look_ahead == 2 else 24)
  for pair in PAIRS:
    dec = beam_cpu.CpuBeamSearch(model, crp_alpha=pair[0], transition_bias=pair[1])
    om = uis_oracle.OracleModel(with_pair(small, pair))
    for x in xs:
      want = uis_oracle.predict_single(om, x, beam_size=5, look_ahead=look_ahead, test_iteration=2)
      assert dec.decode(x, 5, look_ahead, 2) == want, pair
  assert (model.crp_alpha, model.transition_bias) == (small['crp_alpha'], small['transition_bias'])


def test_cpu_score_overrides_match_model_with_pair(small):
  from uisrnn_b200 import beam_cpu
  base = uisrnn_from_weights(small)
  x = utterances(1, 30)[0]
  lab = np.array([0, 0, 1, 1, 1, 0, 2, 2, 0, 1] * 3, np.int32)
  for pair in PAIRS:
    got = beam_cpu.CpuBeamSearch(base, crp_alpha=pair[0], transition_bias=pair[1]).score(x, lab)
    want = beam_cpu.CpuBeamSearch(uisrnn_from_weights(with_pair(small, pair))).score(x, lab)
    assert got[0] == want[0] and np.array_equal(got[1], want[1]), pair


def test_replay_model_reads_the_pair(small):
  """beam_replay.Model takes the pair from the weights dict: its float64 penalty terms move with it."""
  for pair in PAIRS[1:]:
    m = beam_replay.Model(with_pair(small, pair))
    assert m.alpha == pair[0] and m.log_p0 == np.log(pair[1]) and m.pen_last == np.log(1 - pair[1])


def test_predict_sweep_equals_per_pair_models(small):
  model = uisrnn_from_weights(small)
  args = inference_args(beam_size=5, test_iteration=2)
  xs = utterances(2, 20) + [np.zeros((0, 64))]
  got = model.predict(xs, args, decode_params=PAIRS)
  assert len(got) == len(PAIRS)
  for pair, entry in zip(PAIRS, got):
    ref = uisrnn_from_weights(with_pair(small, pair))
    assert entry == ref.predict(xs, args)
  single = model.predict(xs[0], args, decode_params=PAIRS)
  assert single == [entry[0] for entry in got]
  assert (model.crp_alpha, model.transition_bias) == (small['crp_alpha'], small['transition_bias'])


def test_predict_sweep_with_bounds_and_nbest(small):
  model = uisrnn_from_weights(small)
  args = inference_args(beam_size=5, test_iteration=1)
  xs = utterances(2, 20)
  got = model.predict(xs, args, max_speakers=[2, 3], n_best=3, decode_params=PAIRS[1:3])
  for pair, entry in zip(PAIRS[1:3], got):
    ref = uisrnn_from_weights(with_pair(small, pair))
    assert entry == ref.predict(xs, args, max_speakers=[2, 3], n_best=3)
    assert all(max(max(h) for h in nb.labels) < bound for nb, bound in zip(entry, [2, 3]))
  one = model.predict(xs[1], args, max_speakers=2, n_best=2, decode_params=PAIRS[:2])
  assert len(one) == 2 and all(len(nb.labels) <= 2 for nb in one)


def test_predict_sweep_min_speakers_warns_once(small):
  model = uisrnn_from_weights(small)
  args = inference_args(beam_size=3, test_iteration=1)
  xs = utterances(2, 12)
  with warnings.catch_warnings(record=True) as caught:
    warnings.simplefilter('always')
    model.predict(xs, args, min_speakers=12, decode_params=PAIRS[:2])
  msgs = [str(w.message) for w in caught if 'min_speakers' in str(w.message)]
  assert len(msgs) == 1
  assert re.search(r'\(utterance, pair\) \[\(\d, [01]\)', msgs[0])


def test_score_sweep_equals_per_pair_models(small):
  model = uisrnn_from_weights(small)
  xs = utterances(2, 18)
  ids = [['a', 'b', 'b', 'a', 'c', 'c'] * 3, [5, 5, 5, 7, 7, 5] * 3]
  got = model.score(xs, ids, decode_params=PAIRS)
  frames = model.score(xs, ids, per_frame=True, decode_params=PAIRS)
  one = model.score(xs[0], ids[0], decode_params=PAIRS)
  for c, pair in enumerate(PAIRS):
    ref = uisrnn_from_weights(with_pair(small, pair))
    assert got[c] == ref.score(xs, ids)
    want = ref.score(xs, ids, per_frame=True)
    assert [f.total for f in frames[c]] == [f.total for f in want]
    assert all(np.array_equal(a.increments, b.increments) for a, b in zip(frames[c], want))
    assert one[c] == got[c][0]
  assert len({tuple(row) for row in got}) == len(PAIRS)


@pytest.mark.parametrize('bad, index', [
    ([], None), ((), None), ([(1.0, 0.5), (0.0, 0.5)], 1), ([(1.0, 0.5), (-1.0, 0.5)], 1),
    ([(float('nan'), 0.5)], 0), ([(float('inf'), 0.5)], 0), ([(1.0, 0.5), (1.0, 0.5), (1.0, 0.0)], 2),
    ([(1.0, 1.0)], 0), ([(1.0, float('nan'))], 0), ([(1.0, 0.5), (1.0,)], 1), ([(1.0, 0.5), 'ab'], 1),
    ([(True, 0.5)], 0), ('xy', None), (None, None)])
def test_decode_params_validation(small, bad, index):
  model = uisrnn_from_weights(small)
  args = inference_args(beam_size=3, test_iteration=1)
  xs = utterances(1, 6)
  for call in (lambda: model.predict(xs, args, decode_params=bad), lambda: model.score(xs, [[0] * 6], decode_params=bad)):
    if bad is None:
      call()  # None = no sweep
      continue
    with pytest.raises(ValueError) as err:
      call()
    if index is not None:
      assert 'pair {}'.format(index) in str(err.value)


def test_sweep_symbols_in_header_exports_and_library():
  from uisrnn_b200 import native
  header = open(os.path.join(ROOT, 'include', 'uisrnn_b200.h')).read()
  names = ('uis_predict_sweep', 'uis_predict_device_sweep', 'uis_score_sweep', 'uis_score_device_sweep')
  for name in names:
    assert re.search(r'\bint {}\('.format(name), header), name
    assert name in native.EXPORTS
  assert re.search(r'typedef struct uis_decode_params \{\s*int32_t count;\s*const double\* crp_alpha;'
                   r'.*const double\* transition_bias;.*\} uis_decode_params;', header, re.S)
  assert ctypes.sizeof(native.DecodeParams) == 24
  lib = native.load_library()
  for name in names:
    fn = getattr(lib, name)
    assert fn.argtypes[-1] is ctypes.POINTER(native.DecodeParams)
  assert lib.uis_version() == 7
