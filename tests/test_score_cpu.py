"""score() without a GPU: the CPU decoder's forced trace against the reference's own neg_likelihood
(tests/golden/score_cases.npz) and the float64 rescorer, in total and per frame, label canonicalisation, validation,
per-frame increments, and the new C-ABI symbols.  The per-frame check itself is tested: it must reject a swap of two
increments that the total check accepts, an increment a few ulps past its allowance, and a log table cut at 4096
entries."""
import ctypes
import os

import numpy as np
import pytest

from beam_replay import INC_RTOL, PathScores, frame_share, path_score, ulp32
from helpers import GOLDEN, ROOT, load_weights, uisrnn_from_weights


def score_cases():
  """The fixture's cases: name, x (float64 rows), labels, model, score (the reference's total) and frames (its float32
  per-frame losses).  The two long cases store synth_utt arguments instead of rows; they are regenerated here and
  cast to float32 as tools/make_score_golden.py casts them."""
  from uisrnn_b200.synth import synth_utt
  g = np.load(os.path.join(GOLDEN, 'score_cases.npz'))
  toy = np.load(os.path.join(GOLDEN, 'toy_test.npz'))
  off = np.concatenate([[0], np.cumsum(toy['lengths'])])
  cases = []
  for name in g['names']:
    u = int(g[name + '_toy_u'])
    if name + '_synth' in g:
      seed, n, dim, n_spk, noise = g[name + '_synth']
      x = synth_utt(int(seed), n_frames=int(n), dim=int(dim), n_spk=int(n_spk), noise=float(noise))[0]
      x = x.astype(np.float32)
    else:
      x = toy['x'][off[u]:off[u + 1]] if u >= 0 else g[name + '_x']
    cases.append(dict(name=str(name), x=np.asarray(x, np.float64), labels=g[name + '_labels'],
                      model=str(g[name + '_model']), score=float(g[name + '_score']), frames=g[name + '_frames']))
  return cases


CASES = score_cases()
# the toy model (hidden 512) runs slowly on the CPU: a few of its utterances, every small-model case
CPU_CASES = [c for c in CASES if not c['name'].startswith('toy_') or c['name'].endswith(('_0', '_7', '_24'))]

_MODELS = {}


def model(name):
  if name not in _MODELS:
    _MODELS[name] = uisrnn_from_weights(load_weights(name))
  return _MODELS[name]


def check_case(got, case):
  want = case['score']
  if np.isinf(want):
    assert got == want
    return
  assert abs(got - want) <= 1e-5 * abs(want), (case['name'], got, want)
  ps = path_score(load_weights(case['model']), [case['x']], [case['labels']])
  assert ps.share([got])[0] <= 1, (case['name'], got, ps.score[0])


@pytest.mark.parametrize('case', CPU_CASES, ids=[c['name'] for c in CPU_CASES])
def test_cpu_score_matches_reference(case):
  check_case(model(case['model']).score(case['x'], case['labels']), case)


def test_label_names_do_not_matter():
  case = next(c for c in CASES if c['name'] == 's_singletons')
  m = model(case['model'])
  lab = case['labels']
  want = m.score(case['x'], lab)
  perm = np.random.default_rng(3).permutation(lab.max() + 1) + 7
  assert m.score(case['x'], perm[lab]) == want
  assert m.score(case['x'], ['spk%d' % v for v in perm[lab]]) == want
  assert m.score(case['x'], [int(v) for v in lab]) == want
  assert m.score([case['x']], [perm[lab]]) == [want]


def test_per_frame_increments_sum_to_total():
  case = next(c for c in CASES if c['name'] == 's_many')
  fs = model(case['model']).score(case['x'], case['labels'], per_frame=True)
  assert fs.increments.dtype == np.float32 and len(fs.increments) == len(case['x'])
  s = np.float32(0)
  for v in fs.increments:
    s = np.float32(s + v)
  assert float(s) == fs.total


def test_validation_and_empty():
  case = next(c for c in CASES if c['name'] == 's_one_speaker')
  m = model(case['model'])
  x, lab = case['x'], case['labels']
  with pytest.raises(ValueError):
    m.score(x, lab[:-1])
  with pytest.raises(ValueError):
    m.score(x[:, :-1], lab)
  with pytest.raises(TypeError):
    m.score((x,), [lab])
  with pytest.raises(ValueError):
    m.score([x, x], [lab])
  assert m.score(x[:0], []) == 0.0
  assert m.score([x[:0], x], [[], lab]) == [0.0, m.score(x, lab)]


def test_score_symbols_are_exported():
  import __graft_entry__ as ge
  ge.build()
  from uisrnn_b200 import native
  lib = native.load_library()
  assert native.UIS_ABI_VERSION == 7
  for name in ('uis_score', 'uis_score_device'):
    assert name in native.EXPORTS and hasattr(lib, name)
  assert lib.uis_score.argtypes[5] is ctypes.POINTER(ctypes.c_float)
  header = open(os.path.join(ROOT, 'include', 'uisrnn_b200.h')).read()
  assert 'int uis_score(' in header and 'int uis_score_device(' in header


# ---- per frame

_RESCORED = {}


def rescored(model_name):
  """{case name: (float64 increments, Gaussian terms)} of every case of one model, one batched rescore."""
  if model_name not in _RESCORED:
    cases = [c for c in CASES if c['model'] == model_name]
    ps = path_score(load_weights(model_name), [c['x'] for c in cases], [c['labels'] for c in cases], per_frame=True)
    _RESCORED[model_name] = {c['name']: (i, g) for c, i, g in zip(cases, ps.frame_inc, ps.frame_gauss)}
  return _RESCORED[model_name]


def fp32_sum(frames):
  """The fp32 running sum of per-frame increments, in frame order (np.add.accumulate adds sequentially)."""
  f = np.asarray(frames, np.float32)
  return np.float32(np.add.accumulate(f)[-1]) if len(f) else np.float32(0)


@pytest.mark.parametrize('model_name', sorted({c['model'] for c in CASES}))
def test_reference_frames_within_rescore_allowance(model_name):
  """The reference's own per-frame losses lie within the per-frame allowance of the float64 rescore, and add up to
  its totals.  (Worst share measured: 0.53 of the allowance, s_alternating.)"""
  worst = (0.0, None)
  for c in (c for c in CASES if c['model'] == model_name):
    inc, gauss = rescored(model_name)[c['name']]
    share = frame_share(c['frames'], inc, gauss)
    assert share.max() <= 1, (c['name'], int(np.argmax(share)), share.max())
    assert float(fp32_sum(c['frames'])) == c['score'], c['name']
    worst = max(worst, (float(share.max()), c['name']))
  print('%s: worst per-frame share of the reference %.3g (%s)' % (model_name, *worst))


@pytest.mark.parametrize('case', CPU_CASES, ids=[c['name'] for c in CPU_CASES])
def test_cpu_per_frame_matches_reference_bits(case):
  """CpuBeamSearch.score runs the reference's arithmetic frame by frame: its per-frame increments are the reference's
  bits (measured on every case), and so is the total."""
  fs = model(case['model']).score(case['x'], case['labels'], per_frame=True)
  assert np.array_equal(fs.increments.view(np.uint32), case['frames'].view(np.uint32)), \
      int(np.argmax(fs.increments.view(np.uint32) != case['frames'].view(np.uint32)))
  assert fs.total == case['score']


def case_named(name):
  return next(c for c in CASES if c['name'] == name)


def test_per_frame_check_rejects_a_swap_the_total_accepts():
  """Two increments of one utterance swapped (a term written to another frame's row): the fp32 total moves by
  reassociation only and stays within the total allowance; the per-frame check fails at both frames."""
  c = case_named('s_many')
  inc, gauss = rescored(c['model'])[c['name']]
  f = c['frames'].copy()
  i, j = 10, 57
  assert abs(f[i] - f[j]) > 1e-3 * abs(f[i])
  f[[i, j]] = f[[j, i]]
  ps = path_score(load_weights(c['model']), [c['x']], [c['labels']])
  assert ps.share([fp32_sum(f)])[0] <= 1
  share = frame_share(f, inc, gauss)
  assert share[i] > 1 and share[j] > 1 and np.sum(share > 1) == 2


def test_per_frame_check_rejects_four_ulps_past_the_allowance():
  c = case_named('s_singletons')
  inc, gauss = rescored(c['model'])[c['name']]
  assert frame_share(c['frames'], inc, gauss).max() <= 1
  for t in (0, 1, 31, len(inc) - 1):
    edge = inc[t] + ulp32(inc[t]) + INC_RTOL * gauss[t]  # the allowance's upper end
    f = c['frames'].copy()
    f[t] = np.nextafter(np.nextafter(np.nextafter(np.nextafter(np.float32(edge), np.float32(np.inf)),
                                                   np.float32(np.inf)), np.float32(np.inf)), np.float32(np.inf))
    share = frame_share(f, inc, gauss)
    assert share[t] > 1 and np.sum(share > 1) == 1, t


def test_per_frame_check_rejects_a_log_table_cut_at_4096():
  """s_alternating turns at every frame: the increments past turn 4095 recomputed with log(min(turns, 4095) + alpha)
  for the ddCRP denominator -- what a reader of a 4096-entry table that was not regrown gets -- fail per frame; the
  earlier frames are unchanged and pass."""
  c = case_named('s_alternating')
  alpha = float(load_weights(c['model'])['crp_alpha'])
  inc, gauss = rescored(c['model'])[c['name']]
  turns = np.arange(len(c['labels']))  # turns before each frame: every frame opens or moves to a cluster
  f = c['frames'].astype(np.float64)
  past = turns > 4095
  f[past] += np.log(4095 + alpha) - np.log(turns[past] + alpha)
  f = f.astype(np.float32)
  share = frame_share(f, inc, gauss)
  assert np.all(share[~past] <= 1) and np.all(share[past] > 1), (share[past].min(), int(past.sum()))
