"""Latency modes of the beam kernel for few utterances.  Cluster mode: a thread-block cluster of 2/4/8 CTAs per
utterance, every weight matrix split by k-tiles, partial sums exchanged through distributed shared memory.
Stationary-weights mode (cluster=32): 32 CTAs per utterance keep their rows of the weights in shared memory and
exchange results through the shared slot pool with group barriers.  The labels must be those of the reference
(golden) and of the one-CTA-per-utterance path.  Scores, hidden states and running means of both modes are pinned
through the debug taps in test_gpu_latency_modes.py."""
import numpy as np
import pytest

from helpers import GOLDEN, load_weights, toy_utterances

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(180, method='thread')]


@pytest.fixture(scope='module')
def toy_model():
  from uisrnn_b200 import native as nat
  return nat.NativeModel(load_weights('model_toy100.npz'))


@pytest.mark.parametrize('cluster', [2, 4, 8])
def test_forced_cluster_sizes_reproduce_reference_labels(toy_model, cluster):
  xs, labs = toy_utterances()
  xs, labs = xs[:6], labs[:6]
  got = toy_model.predict(xs, cluster=cluster)
  st = toy_model.stats()
  assert st['cluster'] == cluster and st['lanes'] == 1 and st['ctas'] == 6 * cluster
  for i, (g, want) in enumerate(zip(got, labs)):
    assert g.tolist() == want.tolist(), 'utterance %d' % i
  assert st['beam_steps'] == 2 * sum(len(x) for x in xs)      # the replicas of a cluster are counted once


def test_auto_choice_and_opt_out(toy_model):
  xs, labs = toy_utterances()
  one = toy_model.predict([xs[3]])
  assert toy_model.stats()['cluster'] == 32 and toy_model.stats()['ctas'] == 32   # stationary weights: U * 32 <= #SMs
  four = toy_model.predict(xs[:6])
  assert toy_model.stats()['cluster'] == 4 and toy_model.stats()['ctas'] == 24     # 6 utterances: clusters of 4
  assert [f.tolist() for f in four] == [l.tolist() for l in labs[:6]]
  off = toy_model.predict([xs[3]], cluster=-1)
  assert toy_model.stats()['cluster'] == 1 and toy_model.stats()['ctas'] == 1
  assert one[0].tolist() == off[0].tolist() == labs[3].tolist()
  toy_model.predict(xs * 3)                                   # 75 utterances: more than half the SMs
  assert toy_model.stats()['cluster'] == 1
  toy_model.predict(xs * 2)                                   # 50 utterances: pairs of CTAs
  assert toy_model.stats()['cluster'] == 2


def test_ragged_empty_and_more_utterances_than_clusters(toy_model):
  from uisrnn_b200.synth import synth_utt
  xs = [synth_utt(4000 + i, n_frames=n)[0] for i, n in enumerate([37, 1, 64, 2, 90, 5, 23])]
  xs.insert(2, np.zeros((0, 256)))
  want = toy_model.predict(xs, cluster=-1)
  got = toy_model.predict(xs, cluster=4, n_ctas=8)            # 2 clusters take 8 utterances in turn
  assert toy_model.stats()['ctas'] == 8
  assert [g.tolist() for g in got] == [w.tolist() for w in want]
  got = toy_model.predict(xs, cluster=2, beam_size=3, test_iteration=3)
  want = toy_model.predict(xs, cluster=-1, beam_size=3, test_iteration=3)
  assert [g.tolist() for g in got] == [w.tolist() for w in want]


def test_wide_beam_needs_several_passes_per_step(toy_model):
  """beam 30 -> up to 30 distinct source states per step = three 12-column passes, each with its exchanges."""
  from uisrnn_b200.synth import synth_utt
  xs = [synth_utt(4100 + i, n_frames=60, n_spk=4)[0] for i in range(2)]
  got = toy_model.predict(xs, cluster=4, beam_size=30, kcap=16)
  want = toy_model.predict(xs, cluster=-1, beam_size=30, kcap=16)
  assert [g.tolist() for g in got] == [w.tolist() for w in want]


def test_synth500_in_cluster_mode(toy_model):
  from uisrnn_b200.synth import synth_utt
  g = np.load(GOLDEN + '/synth500.npz')
  xs = [synth_utt(int(s))[0] for s in g['seeds']]
  got = toy_model.predict(xs, cluster=4)
  for o, want in zip(got, g['labels']):
    assert o.tolist() == want.tolist()


def test_stationary_weights_mode_reproduces_reference_labels(toy_model):
  """cluster=32: all 25 toy utterances through groups of 32 CTAs (4 groups on a 132-SM device take them in turn)."""
  xs, labs = toy_utterances()
  got = toy_model.predict(xs, cluster=32)
  st = toy_model.stats()
  assert st['cluster'] == 32 and st['lanes'] == 1 and st['ctas'] == 128 and st['engine'] == 1
  for i, (g, want) in enumerate(zip(got, labs)):
    assert g.tolist() == want.tolist(), 'utterance %d' % i
  assert st['beam_steps'] == 2 * sum(len(x) for x in xs)      # the replicas of a group are counted once


def test_stationary_weights_mode_on_500_frame_goldens_and_ragged_lists(toy_model):
  from uisrnn_b200.synth import synth_utt
  g = np.load(GOLDEN + '/synth500.npz')
  xs = [synth_utt(int(s))[0] for s in g['seeds']]
  got = toy_model.predict(xs)                                 # 2 utterances: chosen automatically
  assert toy_model.stats()['cluster'] == 32 and toy_model.stats()['ctas'] == 64
  for o, want in zip(got, g['labels']):
    assert o.tolist() == want.tolist()
  xs = [synth_utt(4000 + i, n_frames=n)[0] for i, n in enumerate([37, 1, 64, 2, 90, 5, 23])]
  xs.insert(2, np.zeros((0, 256)))
  want = toy_model.predict(xs, cluster=-1)
  got = toy_model.predict(xs, cluster=32, n_ctas=64)          # 2 groups take 8 utterances in turn
  assert toy_model.stats()['ctas'] == 64
  assert [o.tolist() for o in got] == [w.tolist() for w in want]
  got = toy_model.predict(xs[:3], cluster=32, beam_size=30, kcap=16, test_iteration=3)   # 3 passes of 12 columns per step
  want = toy_model.predict(xs[:3], cluster=-1, beam_size=30, kcap=16, test_iteration=3)
  assert [o.tolist() for o in got] == [w.tolist() for w in want]
