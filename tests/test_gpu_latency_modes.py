"""The latency modes of the look_ahead-1 beam kernel -- cluster mode (cluster=2/4/8: the CTAs of a thread-block cluster
split every weight matrix by k-tiles and all-reduce the partial sums through distributed shared memory) and
stationary-weights mode (cluster=32: 32 CTAs keep the weights in shared memory, split each product by rows and share
one slot pool in global memory) -- pinned at score and state level through the debug taps: the per-step winners and
scores of the traced utterance (1e-5 relative, near-ties at the beam cut-off tolerated by compare_trace), the final
scores of every utterance (1e-5 relative), the running means and hidden states of the best hypothesis (1e-5 absolute)
and its block counts (exact).  Labels alone miss most of what can go wrong in these modes: a k-tile counted twice, an
exchange buffer reused a round early or a stale read of a slot another CTA wrote move values by small amounts.

Every test asserts the mode the call ran in (`stats()['cluster']`), so that a fall-back to the one-CTA kernel fails.
The last tests trace every lane of a multi-lane CTA (tensor-core engine, FFMA with two lanes), whose column bases and
pool strides lane 0 never exercises."""
import os

import numpy as np
import pytest

from helpers import GOLDEN, compare_trace, load_weights, rel_err, toy_utterances, uis_oracle
from test_gpu_large_models import large_model

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method='thread')]

SCORE_RTOL = 1e-5
STATE_ATOL = 1e-5
MODES = [2, 4, 8, 32]
# (beam_size, test_iteration, kcap): beam 30 takes three 12-column passes per step (several exchange rounds each) and
# needs kcap 16 to fit shared memory; kcap 64 leaves room for every cluster the untrained model opens
CONFIGS = [(1, 1, 64), (4, 1, 64), (10, 2, 64), (10, 3, 64), (30, 1, 16)]
LENGTHS = (1, 2, 37, 120)
LANE_LENGTHS = (41, 23, 36, 17, 48, 29)


def untrained_weights(H, D, seed):
  """An untrained model as in test_gpu_large_models (sigma2 0.003, transition_bias 0.3) with h0 scaled by 3, so that
  its decodes open many clusters."""
  w = large_model(H, D, 1, seed)
  w['h0'] = 3.0 * w['h0']
  return w


def model_weights(name):
  if name == 'toy':
    return load_weights('model_toy100.npz')
  if name == 'untrained':
    return untrained_weights(512, 256, 71)
  assert name == 'untrained256'
  return untrained_weights(256, 128, 72)


# Seeds of the synthetic utterances.  Picked so that every decode of 37 frames or more shows at least three labels,
# that no hypothesis of the beam-30 decodes exceeds kcap 16 nor one of the (256, 128) model's decodes the tensor-core
# engine's default kcap 16, and that no exact tie at the beam cut-off changes the trace: the kernels keep the
# tied candidate with the lower flat index, the reference's unstable sort may keep the other one, and from there on
# the two searches follow different hypotheses.
FRESH_SEEDS = {'toy': (6300, 21000, 22005, 6305), 'untrained': (6400, 21300, 22300, 23301)}
LANE_SEEDS = {'toy': (6500, 6501, 6502, 6503, 6504, 6505), 'untrained256': (7011, 6833, 6962, 23603, 24601, 25603)}


def inputs(name, lengths, seeds):
  """Five speakers changing every ~3 frames, so that even beam 1 opens several clusters."""
  from uisrnn_b200.synth import synth_utt
  D = 128 if name == 'untrained256' else 256
  return [synth_utt(s, n_frames=n, dim=D, n_spk=5, mean_run=3, noise=0.02)[0] for s, n in zip(seeds, lengths)]


def fresh_inputs(name):
  return inputs(name, LENGTHS, FRESH_SEEDS[name])


def lane_inputs(name):
  return inputs(name, LANE_LENGTHS, LANE_SEEDS[name])


_ORACLE_MODELS = {}


def _oracle_job(job):
  """(model name, 'fresh' | 'lanes', utterance index, beam, test_iteration) -> (labels, record)."""
  name, batch, i, beam, titer = job
  if name not in _ORACLE_MODELS:
    _ORACLE_MODELS[name] = uis_oracle.OracleModel(model_weights(name))
  x = (fresh_inputs if batch == 'fresh' else lane_inputs)(name)[i]
  rec = {}
  labels = uis_oracle.predict_single(_ORACLE_MODELS[name], x, beam_size=beam, look_ahead=1, test_iteration=titer,
                                     record=rec)
  return labels, rec


def oracle_jobs():
  jobs = [(name, 'fresh', i, beam, titer) for name in ('toy', 'untrained') for beam, titer, _ in CONFIGS
          for i in range(len(LENGTHS))]
  jobs += [(name, 'lanes', i, 10, 2) for name in ('toy', 'untrained256') for i in range(len(LANE_LENGTHS))]
  return jobs


@pytest.fixture(scope='module')
def oracle():
  """Every oracle decode of the module, keyed by job.  A single BLAS thread: the oracle's products are small, and
  threads spun up for each of them make it many times slower."""
  from threadpoolctl import threadpool_limits
  with threadpool_limits(limits=1):
    return {job: _oracle_job(job) for job in oracle_jobs()}


@pytest.fixture(scope='module')
def native():
  from uisrnn_b200 import native as nat
  nat.load_library()
  return nat


_MODELS = {}


def native_model(native, name):
  if name not in _MODELS:
    _MODELS[name] = native.NativeModel(model_weights(name))
  return _MODELS[name]


def check_traced(dbg, rec):
  """Per-step winners and scores, then the best hypothesis's running means, hidden states and block counts."""
  compare_trace(dbg['win'], dbg['score'], dbg['off'], rec['win'], rec['score'], rec['off'], rtol=SCORE_RTOL)
  assert dbg['best_mean'].shape == rec['final_mean'].shape
  assert dbg['best_hidden'].shape == rec['final_hidden'].shape
  assert np.max(np.abs(dbg['best_mean'] - rec['final_mean'])) < STATE_ATOL
  assert np.max(np.abs(dbg['best_hidden'] - rec['final_hidden'])) < STATE_ATOL
  assert np.array_equal(dbg['best_blocks'], rec['final_blocks'])


def check_final_scores(dbg, recs):
  """Final scores and cluster count of the best hypothesis of every utterance; None = an empty utterance."""
  for u, rec in enumerate(recs):
    got = dbg['final_scores'][u]
    if rec is None:
      assert np.all(np.isinf(got)) and dbg['final_k'][u] == 0, 'utterance %d' % u
      continue
    nb = len(rec['final_scores'])
    assert rel_err(got[:nb], rec['final_scores']) < SCORE_RTOL, 'utterance %d' % u
    assert np.all(np.isinf(got[nb:])), 'utterance %d' % u
    assert dbg['final_k'][u] == len(rec['final_mean']), 'utterance %d' % u


def check_every_utterance_traced(model, xs, want, kw, check_stats):
  """One call per utterance, each tracing that utterance: labels, final scores of all, the traced one's trace and
  state.  `want` holds (labels, record) per utterance, None for an empty one."""
  for u, x in enumerate(xs):
    got, dbg = model.predict(xs, trace_utt=u, **kw)
    check_stats(model.stats())
    for v, (g, w) in enumerate(zip(got, want)):
      assert g.tolist() == (w[0] if w else []), 'traced %d: labels of utterance %d' % (u, v)
    check_final_scores(dbg, [w[1] if w else None for w in want])
    if want[u]:
      check_traced(dbg, want[u][1])


def stats_check(mode, ctas=None):
  def check(st):
    assert st['cluster'] == mode and st['lanes'] == 1 and st['engine'] == 1
    if ctas is not None:
      assert st['ctas'] == ctas
  return check


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('idx', [0, 1])
def test_reference_trace(native, mode, idx):
  """Per-step winners and scores of the reference's own trace; running means and hidden states of its best
  hypothesis."""
  model = native_model(native, 'toy')
  xs, _ = toy_utterances()
  g = np.load(os.path.join(GOLDEN, 'toy_trace.npz'))
  got, dbg = model.predict([xs[idx]], trace_utt=0, cluster=mode)
  assert model.stats()['cluster'] == mode
  assert got[0].tolist() == g['u%d_labels' % idx].tolist()
  compare_trace(dbg['win'], dbg['score'], dbg['off'], g['u%d_win' % idx], g['u%d_score' % idx], g['u%d_off' % idx],
                rtol=SCORE_RTOL)
  assert rel_err(dbg['final_scores'][0], g['u%d_final_scores' % idx]) < SCORE_RTOL
  assert np.max(np.abs(dbg['best_hidden'] - g['u%d_final_hidden' % idx])) < STATE_ATOL
  assert np.max(np.abs(dbg['best_mean'] - g['u%d_final_mean' % idx])) < STATE_ATOL
  assert np.array_equal(dbg['best_blocks'], g['u%d_final_blocks' % idx])


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('beam,titer,kcap', CONFIGS)
@pytest.mark.parametrize('name', ['toy', 'untrained'])
def test_fresh_inputs_against_oracle(native, oracle, name, beam, titer, kcap, mode):
  """Utterances of 1, 2, 37 and 120 frames decoded together, each one traced in turn; the labels with taps must be
  those without."""
  model = native_model(native, name)
  xs = fresh_inputs(name)
  want = [oracle[(name, 'fresh', i, beam, titer)] for i in range(len(xs))]
  for x, (labels, _) in zip(xs, want):
    if len(x) >= 37:
      assert len(set(labels)) >= 3, 'trivial decode: %s' % labels
  kw = dict(beam_size=beam, test_iteration=titer, kcap=kcap, cluster=mode)
  plain = model.predict(xs, **kw)
  stats_check(mode)(model.stats())
  assert [p.tolist() for p in plain] == [w[0] for w in want]
  check_every_utterance_traced(model, xs, want, kw, stats_check(mode))


@pytest.mark.parametrize('mode', MODES)
def test_one_cluster_decodes_utterances_in_turn(native, oracle, mode):
  """One cluster / group takes a ragged batch with an empty utterance in turn (longest first): what a new utterance
  resets -- the replicated lane state, the exchange-buffer parity, the group barrier's epoch, the shared slot pool --
  shows in the trace of the second and third utterance it decodes."""
  model = native_model(native, 'toy')
  fresh = fresh_inputs('toy')
  xs = [fresh[2], np.zeros((0, 256)), fresh[3], fresh[1]]
  want = [oracle[('toy', 'fresh', i, 10, 2)] if i is not None else None for i in (2, None, 3, 1)]
  check_every_utterance_traced(model, xs, want, dict(beam_size=10, test_iteration=2, cluster=mode, n_ctas=mode),
                               stats_check(mode, ctas=mode))


def test_taps_keep_the_automatic_plan(native):
  """A traced call plans the kernel an untraced one does: stationary weights for one utterance, clusters of 4 for
  six (as in test_gpu_cluster.py::test_auto_choice_and_opt_out)."""
  model = native_model(native, 'toy')
  xs, labs = toy_utterances()
  got, dbg = model.predict([xs[3]], trace_utt=0)
  assert model.stats()['cluster'] == 32 and model.stats()['ctas'] == 32
  assert got[0].tolist() == labs[3].tolist() and len(dbg['off']) == 2 * len(xs[3]) + 1
  got, dbg = model.predict(xs[:6], trace_utt=5)
  assert model.stats()['cluster'] == 4 and model.stats()['ctas'] == 24
  assert [g.tolist() for g in got] == [l.tolist() for l in labs[:6]] and len(dbg['off']) == 2 * len(xs[5]) + 1


LANE_CASES = {
    # name: (model, engine, lanes): one CTA's worth of utterances, so that every lane is traced once
    'tc-512x256': ('toy', 2, 6),
    'tc-256x128': ('untrained256', 2, 6),
    'ffma-lanes2': ('toy', 1, 2),
}


@pytest.mark.parametrize('case', list(LANE_CASES))
def test_every_lane_of_a_cta_traced(native, oracle, case):
  name, engine, lanes = LANE_CASES[case]
  model = native_model(native, name)
  xs = lane_inputs(name)[:lanes]
  want = [oracle[(name, 'lanes', i, 10, 2)] for i in range(lanes)]
  for x, (labels, _) in zip(xs, want):
    assert len(set(labels)) >= 3, 'trivial decode: %s' % labels

  def check(st):
    assert st['engine'] == engine and st['lanes'] == lanes and st['ctas'] == 1 and st['cluster'] == 1

  check_every_utterance_traced(model, xs, want, dict(engine=engine, lanes=lanes, n_ctas=1), check)
