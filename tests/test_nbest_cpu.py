"""N-best predict() without a GPU: the CPU decoder's N best hypotheses against the reference's own search (every final
rank back-tracked through its recorded winners, and the final beams of the speaker-bounds fixture), argument checking,
return types, and the ctypes signatures of the N-best entry points."""
import ctypes
import os

import numpy as np
import pytest

from beam_replay import backtrack, ulp32
from helpers import ROOT, inference_args, load_weights, uisrnn_from_weights
from test_beam_replay_cpu import GOLDEN_CASES
from test_speaker_bounds_cpu import CASES as BOUND_CASES

# the reference's toy model (hidden 512) decodes slowly on the CPU: its traced utterances run at k = 3 only
CPU_CASES = [c for c in GOLDEN_CASES if not c['name'].startswith('bounds_')]
CPU_IDS = [c['name'] for c in CPU_CASES]


def expected_from_trace(case, k):
  """(labels, scores, clusters) of the first k qualifying final ranks, from the reference's winner records."""
  win, off, score = case['win'], case['off'], case['score']
  n, tn = len(case['x']), len(case['x']) * case['test_iteration']
  finals = int(off[-1] - off[-2])
  clusters = [max(backtrack(win, off, tn, r)) + 1 for r in range(finals)]
  final_scores = score[int(off[-2]):int(off[-1])].astype(np.float64)
  from uisrnn_b200.beam_cpu import nbest_ranks
  ranks = nbest_ranks(clusters, case.get('min_speakers', 0), k)
  return ranks, [backtrack(win, off, n, r) for r in ranks], final_scores, clusters


def check_nbest(got, ranks, rank_labels, final_scores, clusters):
  """got = (labels, scores, clusters) of the decoder.  A hypothesis may stand in for its neighbour rank where the two
  fp32 scores differ by at most one ulp (the reference sorts with an unstable sort)."""
  labels, scores, ks = got
  assert len(labels) == len(scores) == len(ks) == len(ranks)
  for j, r in enumerate(ranks):
    want = float(final_scores[r])
    assert abs(scores[j] - want) <= 1e-5 * max(1.0, abs(want)), (j, scores[j], want)
    if labels[j] != rank_labels[j]:
      near = [q for q in (r - 1, r + 1) if 0 <= q < len(final_scores) and
              abs(final_scores[q] - final_scores[r]) <= float(ulp32(final_scores[r]))]
      assert near, 'hypothesis %d differs from final rank %d without a tie' % (j, r)
    assert ks[j] == clusters[r] or labels[j] != rank_labels[j]


def decoder(case):
  from uisrnn_b200 import beam_cpu
  return beam_cpu.CpuBeamSearch(uisrnn_from_weights(load_weights(case['model'])))


@pytest.mark.parametrize('case', CPU_CASES, ids=CPU_IDS)
def test_cpu_nbest_matches_reference_trace(case):
  dec = decoder(case)
  ks = (3,) if case['model'] == 'model_toy100.npz' else sorted({1, 3, case['beam_size']})
  for k in ks:
    k = min(k, case['beam_size'])
    got = dec.decode(case['x'], case['beam_size'], case['look_ahead'], case['test_iteration'], n_best=k)
    ranks, rank_labels, final_scores, clusters = expected_from_trace(case, k)
    check_nbest(got, ranks, rank_labels, final_scores, clusters)
    assert got[0][0] == case['labels'].tolist()  # hypothesis 0 = the reference's labels


BOUND_CPU = [c for c in BOUND_CASES if c['model'] != 'model_toy100.npz']


@pytest.mark.parametrize('case', BOUND_CPU, ids=[c['name'] for c in BOUND_CPU])
def test_cpu_nbest_matches_bounded_final_beam(case):
  """Speaker bounds: the N best are the first final ranks with min_speakers clusters (rank 0 alone when none)."""
  from uisrnn_b200.beam_cpu import nbest_ranks
  dec = decoder(case)
  finals = int(np.isfinite(case['final_scores']).sum())
  final_k = [int(v) for v in case['final_k'][:finals]]
  for k in sorted({1, 3, case['beam_size']}):
    got = dec.decode(case['x'], case['beam_size'], case['look_ahead'], case['test_iteration'], case['max_speakers'],
                     case['min_speakers'], n_best=k)
    ranks = nbest_ranks(final_k, case['min_speakers'], k)
    assert ranks[0] == int(case['chosen'])
    check_nbest(got, ranks, [case['final_traces'][r].tolist() for r in ranks], case['final_scores'].astype(np.float64),
                final_k)
    assert got[0][0] == case['labels'].tolist()
  if case['name'] == 's_min_fallback':
    assert len(got[0]) == 1 and got[2][0] < case['min_speakers']


def test_uisrnn_predict_nbest_cpu_types_and_validation():
  from uisrnn_b200.uisrnn import NBest
  case = {c['name']: c for c in BOUND_CASES}['s_b10_la1_t2']
  model = uisrnn_from_weights(load_weights(case['model']))
  args = inference_args(case['beam_size'], case['look_ahead'], case['test_iteration'])
  x = case['x']
  plain = model.predict(x, args)
  one = model.predict(x, args, n_best=3)
  assert isinstance(one, NBest) and len(one.labels) == 3 and one.labels[0] == plain
  assert all(isinstance(v, float) for v in one.scores) and all(isinstance(v, int) for v in one.speakers)
  assert one.scores == sorted(one.scores)
  many = model.predict([x, x[:7], x[:0]], args, n_best=2, max_speakers=[2, 0, 0])
  assert isinstance(many, list) and all(isinstance(o, NBest) for o in many)
  assert many[0].labels[0] == model.predict(x, args, max_speakers=2) and max(many[0].speakers) <= 2
  assert many[1].labels[0] == model.predict(x[:7], args)
  assert many[2] == NBest([], [], [])  # an empty sequence: no hypothesis
  assert model.predict_single(x, args, n_best=1) == NBest([plain], one.scores[:1], one.speakers[:1])
  for bad in (0, -1, args.beam_size + 1, 2.0, True, '3', [2]):
    with pytest.raises(ValueError):
      model.predict(x, args, n_best=bad)
    with pytest.raises(ValueError):
      model.predict([x], args, n_best=bad)


def test_parallel_predict_nbest_cpu():
  from uisrnn_b200.uisrnn import parallel_predict
  case = {c['name']: c for c in BOUND_CASES}['s_b10_la1_t2']
  model = uisrnn_from_weights(load_weights(case['model']))
  args = inference_args(case['beam_size'], case['look_ahead'], case['test_iteration'])
  xs = [case['x'], case['x'][:9]]
  assert parallel_predict(model, xs, args, num_processes=2, n_best=3) == model.predict(xs, args, n_best=3)
  with pytest.raises(ValueError):
    parallel_predict(model, xs, args, num_processes=2, n_best=0)


def test_nbest_entry_point_signatures():
  import __graft_entry__ as ge
  ge.build()
  from uisrnn_b200 import native
  lib = native.load_library()
  for name in ('uis_predict_nbest', 'uis_predict_device_nbest'):
    assert name in native.EXPORTS and hasattr(lib, name)
  header = open(os.path.join(ROOT, 'include', 'uisrnn_b200.h')).read()
  for name in ('uis_predict_nbest', 'uis_predict_device_nbest'):
    decl = header[header.index('int ' + name + '('):]
    decl = decl[:decl.index(';')]
    assert decl.rstrip(')').endswith('const uis_nbest_out* out'), decl
    assert 'const int32_t* max_speakers, const int32_t* min_speakers, int32_t n_best' in decl
  assert ctypes.sizeof(native.NBestOut) == 5 * ctypes.sizeof(ctypes.c_void_p)
