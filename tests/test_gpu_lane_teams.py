"""Lane counts of the look_ahead-1 beam kernel that bench.py's workload does not run.  Each lane's selection phases
run on a team of NW / lanes consumer warps: one warp at 5 and 7 lanes, two warps with named team barriers at 3 lanes
(two warps own no lane on the tensor-core engine), the whole consumer set at 1 lane.  Every such count must give the
reference's labels on the 500-frame goldens, and, with n_best and speaker bounds, the outputs of the same engine run
one lane per CTA, bit for bit; plane 0 must be the FFMA engine's labels."""
import numpy as np
import pytest

from helpers import GOLDEN, load_weights

pytestmark = pytest.mark.gpu

# (engine, lanes, kcap): kcap 12 lets 7 tensor-core lanes of beam 10 fit in shared memory
REFERENCE = [(2, 3, 16), (2, 5, 16), (2, 7, 12), (1, 3, 16)]
# (engine, lanes, beam_size, kcap, n_best); beam 64 runs with max_speakers <= kcap = 2 so that three lanes fit
NBEST = [(2, 3, 10, 12, 4), (2, 5, 10, 12, 4), (2, 7, 10, 12, 4), (1, 3, 10, 12, 4), (2, 3, 64, 2, 8), (1, 3, 64, 2, 8)]


def engine_kw(engine):
  return dict(engine=engine, cluster=-1) if engine == 1 else dict(engine=engine)


@pytest.fixture(scope='module')
def toy_model():
  from uisrnn_b200 import native
  native.load_library()
  return native.NativeModel(load_weights('model_toy100.npz'))


@pytest.mark.parametrize('engine,lanes,kcap', REFERENCE, ids=['engine%d-lanes%d' % (e, g) for e, g, _ in REFERENCE])
def test_reference_labels_500_frames(toy_model, engine, lanes, kcap):
  """12 golden utterances on one CTA: every lane decodes several utterances in turn."""
  from uisrnn_b200.synth import synth_utt
  xs, want = [], []
  for name in ('synth500_bench', 'synth500'):
    g = np.load(GOLDEN + '/%s.npz' % name)
    xs += [synth_utt(int(s))[0] for s in g['seeds']]
    want += [lab.tolist() for lab in g['labels']]
  got = toy_model.predict(xs, lanes=lanes, n_ctas=1, kcap=kcap, **engine_kw(engine))
  st = toy_model.stats()
  assert st['engine'] == engine and st['lanes'] == lanes and st['ctas'] == 1
  for i, (g, w) in enumerate(zip(got, want)):
    assert g.tolist() == w, 'utterance %d' % i


def batch(beam_size):
  from uisrnn_b200.synth import synth_utt
  xs = [synth_utt(9500 + u, n_frames=50 + 13 * u, n_spk=2 + u % 3, noise=0.06)[0] for u in range(11)]
  if beam_size > 32:
    mx = np.full(len(xs), 2, np.int32)
    mn = np.array([2, 0, 1, 2, 0, 2, 1, 0, 2, 2, 0], np.int32)
  else:
    mx = np.array([0, 3, 2, 0, 4, 1, 0, 3, 2, 0, 4], np.int32)
    mn = np.array([0, 2, 2, 0, 3, 0, 0, 1, 2, 0, 4], np.int32)
  return xs, mx, mn


@pytest.mark.parametrize('engine,lanes,beam_size,kcap,k', NBEST,
                         ids=['engine%d-lanes%d-beam%d' % (e, g, b) for e, g, b, _, _ in NBEST])
def test_nbest_and_bounds_equal_one_lane(toy_model, engine, lanes, beam_size, kcap, k):
  xs, mx, mn = batch(beam_size)
  kw = dict(beam_size=beam_size, test_iteration=2, kcap=kcap, n_ctas=1, n_best=k, max_speakers=mx, min_speakers=mn)
  labels, scores, speakers, count = toy_model.predict(xs, lanes=lanes, **kw, **engine_kw(engine))
  st = toy_model.stats()
  assert st['engine'] == engine and st['lanes'] == lanes
  one = toy_model.predict(xs, lanes=1, **kw, **engine_kw(engine))
  assert toy_model.stats()['lanes'] == 1
  ffma = toy_model.predict(xs, lanes=1, **dict(kw, n_best=None), **engine_kw(1))
  for u in range(len(xs)):
    assert np.array_equal(labels[u], one[0][u]), u
    assert np.array_equal(scores[u].view(np.int32), one[1][u].view(np.int32)), u
    assert np.array_equal(speakers[u], one[2][u]) and count[u] == one[3][u], u
    assert np.array_equal(labels[u][0], ffma[u]), u
    assert count[u] >= 1
