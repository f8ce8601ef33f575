"""score() without a GPU: the CPU decoder's forced trace against the reference's own neg_likelihood
(tests/golden/score_cases.npz) and the float64 rescorer, label canonicalisation, validation, per-frame increments, and
the new C-ABI symbols."""
import ctypes
import os

import numpy as np
import pytest

from beam_replay import path_score
from helpers import GOLDEN, ROOT, load_weights, uisrnn_from_weights


def score_cases():
  g = np.load(os.path.join(GOLDEN, 'score_cases.npz'))
  toy = np.load(os.path.join(GOLDEN, 'toy_test.npz'))
  off = np.concatenate([[0], np.cumsum(toy['lengths'])])
  cases = []
  for name in g['names']:
    u = int(g[name + '_toy_u'])
    x = toy['x'][off[u]:off[u + 1]] if u >= 0 else g[name + '_x']
    cases.append(dict(name=str(name), x=np.asarray(x, np.float64), labels=g[name + '_labels'],
                      model=str(g[name + '_model']), score=float(g[name + '_score'])))
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
