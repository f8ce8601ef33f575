"""Speaker bounds (max_speakers / min_speakers) without a GPU: the bounded oracle against the reference's own search
(tests/golden/speaker_bounds_cases.npz), the CPU decoder against the oracle, argument checking of the public API,
and the ctypes signatures of the bounded entry points."""
import ctypes
import os
import warnings

import numpy as np
import pytest

from helpers import GOLDEN, ROOT, compare_trace, inference_args, load_weights, oracle_model, rel_err, \
    uisrnn_from_weights
import speaker_bounds_oracle as SB


def bound_cases():
  g = np.load(os.path.join(GOLDEN, 'speaker_bounds_cases.npz'))
  out = []
  for name in g['names']:
    name = str(name)
    b, la, t = [int(v) for v in g[name + '_args']]
    mx, mn = [int(v) for v in g[name + '_bounds']]
    out.append(dict(name=name, model=str(g[name + '_model']), x=g[name + '_x'].astype(np.float64), beam_size=b,
                    look_ahead=la, test_iteration=t, max_speakers=mx, min_speakers=mn,
                    **{k: g['{}_{}'.format(name, k)] for k in
                       ('labels', 'unbounded', 'win', 'score', 'off', 'nfinite', 'final_scores', 'final_k',
                        'final_traces', 'chosen')}))
  return out


CASES = bound_cases()
IDS = [c['name'] for c in CASES]


def run_oracle(case, **over):
  kw = dict(beam_size=case['beam_size'], look_ahead=case['look_ahead'], test_iteration=case['test_iteration'],
            max_speakers=case['max_speakers'], min_speakers=case['min_speakers'])
  kw.update(over)
  rec = {}
  labels = SB.predict_single(oracle_model(case['model']), case['x'], record=rec, **kw)
  return labels, rec


def test_fixture_covers_the_issue_matrix():
  args = {(c['model'], c['beam_size'], c['look_ahead'], c['test_iteration']) for c in CASES}
  small = {a[1:] for a in args if a[0] == 'model_small.npz'}
  assert {b for b, _, _ in small} >= {1, 10, 30}
  assert {la for _, la, _ in small} >= {1, 2, 3}
  assert {t for _, _, t in small} >= {1, 2}
  for model in ('model_small_d2.npz', 'model_toy100.npz'):
    assert {a[2] for a in args if a[0] == model} >= {1, 2}
  for c in CASES:
    if c['max_speakers']:  # the bound binds: the unbounded search opens more clusters
      assert c['unbounded'].max() + 1 > c['max_speakers'] and c['labels'].max() < c['max_speakers']
  for model in ('model_small.npz', 'model_toy100.npz'):  # a fallback to rank 0 and a pick further down the final beam
    chosen = [int(c['chosen']) for c in CASES if c['min_speakers'] and c['model'] == model]
    assert min(chosen) == 0 and max(chosen) > 0, model
  # the toy-model min cases run at look_ahead 1: the tensor-core / cluster / stationary-weights kernels take them
  assert all(c['look_ahead'] == 1 for c in CASES if c['min_speakers'] and c['model'] == 'model_toy100.npz')


@pytest.mark.parametrize('case', CASES, ids=IDS)
def test_oracle_reproduces_reference(case):
  labels, rec = run_oracle(case)
  assert labels == case['labels'].tolist()
  compare_trace(rec['win'], rec['score'], rec['off'], case['win'], case['score'], case['off'])
  assert np.array_equal(rec['nfinite'], case['nfinite'])
  assert np.array_equal(rec['final_k'], case['final_k'])
  assert np.array_equal(rec['final_traces'], case['final_traces'])
  assert rec['chosen'] == int(case['chosen'])
  assert rel_err(rec['final_scores'], case['final_scores']) < 1e-5


def test_unbounded_oracle_is_the_plain_oracle():
  from helpers import uis_oracle
  case = CASES[0]
  model = oracle_model(case['model'])
  kw = dict(beam_size=case['beam_size'], look_ahead=case['look_ahead'], test_iteration=case['test_iteration'])
  plain, bounded = {}, {}
  a = uis_oracle.predict_single(model, case['x'], record=plain, **kw)
  b = SB.predict_single(model, case['x'], record=bounded, **kw)
  assert a == b == case['unbounded'].tolist()
  assert np.array_equal(plain['win'], bounded['win']) and np.array_equal(plain['score'], bounded['score'])


def uisrnn_model(name):
  return uisrnn_from_weights(load_weights(name))


def case_args(case):
  return inference_args(case['beam_size'], case['look_ahead'], case['test_iteration'])


@pytest.mark.parametrize('case', [c for c in CASES if c['model'] != 'model_toy100.npz'],
                         ids=[c['name'] for c in CASES if c['model'] != 'model_toy100.npz'])
def test_cpu_decoder_matches_oracle(case):
  from uisrnn_b200 import beam_cpu
  dec = beam_cpu.CpuBeamSearch(uisrnn_model(case['model']))
  labels, k = dec.decode(case['x'], case['beam_size'], case['look_ahead'], case['test_iteration'],
                         case['max_speakers'], case['min_speakers'], return_speakers=True)
  assert labels == case['labels'].tolist()
  assert k == case['final_k'][int(case['chosen'])]


def test_uisrnn_predict_cpu_bounds_and_validation():
  model = uisrnn_model('model_small.npz')
  by_name = {c['name']: c for c in CASES}
  a, b = by_name['s_b10_la1_t2'], by_name['s_min_pick']
  args = case_args(a)
  assert args.beam_size == b['beam_size'] and args.look_ahead == b['look_ahead']
  args.test_iteration = 2
  # int bound: every utterance; per-utterance bounds, one unbounded
  both = model.predict([a['x'], a['x']], args, max_speakers=a['max_speakers'])
  assert both == [a['labels'].tolist()] * 2
  mixed = model.predict([a['x'], a['x']], args, max_speakers=[a['max_speakers'], 0])
  assert mixed[0] == a['labels'].tolist() and mixed[1] == a['unbounded'].tolist()
  assert model.predict(a['x'], args, max_speakers=a['max_speakers']) == a['labels'].tolist()
  assert model.predict([a['x']], args) == [a['unbounded'].tolist()]
  # the fallback warns once, naming the utterance
  fb = by_name['s_min_fallback']
  fargs = case_args(fb)
  with warnings.catch_warnings(record=True) as caught:
    warnings.simplefilter('always')
    out = model.predict([a['x'][:5], fb['x']], fargs, min_speakers=[0, fb['min_speakers']])
  assert out[1] == fb['labels'].tolist()
  msgs = [str(w.message) for w in caught if 'min_speakers' in str(w.message)]
  assert len(msgs) == 1 and '[1]' in msgs[0]
  for bad in (dict(max_speakers=-1), dict(min_speakers=-2), dict(max_speakers=2, min_speakers=3),
              dict(max_speakers=[1, 2, 3]), dict(min_speakers=[1]), dict(max_speakers=2.7),
              dict(min_speakers=[1.0, 2.0]), dict(max_speakers=True)):
    with pytest.raises(ValueError):
      model.predict([a['x'], a['x']], args, **bad)
  with pytest.raises(ValueError):
    model.predict_single(a['x'], args, max_speakers=[2])


def test_parallel_predict_cpu_with_bounds():
  """The CPU device's process pool: per-utterance bounds travel with their utterances."""
  from uisrnn_b200.uisrnn import parallel_predict
  model = uisrnn_model('model_small.npz')
  by_name = {c['name']: c for c in CASES}
  a, fb = by_name['s_b10_la1_t2'], by_name['s_min_fallback']
  out = parallel_predict(model, [a['x'], a['x']], case_args(a), num_processes=2,
                         max_speakers=[a['max_speakers'], 0])
  assert out == [a['labels'].tolist(), a['unbounded'].tolist()]
  with warnings.catch_warnings(record=True) as caught:
    warnings.simplefilter('always')
    out = parallel_predict(model, [a['x'][:5], fb['x']], case_args(fb), num_processes=2,
                           min_speakers=[0, fb['min_speakers']])
  assert out[1] == fb['labels'].tolist()
  assert len([w for w in caught if 'min_speakers' in str(w.message) and '[1]' in str(w.message)]) == 1
  with pytest.raises(ValueError):
    parallel_predict(model, [a['x']], case_args(a), num_processes=2, max_speakers=2.5)


def test_bounded_entry_point_signatures():
  import __graft_entry__ as ge
  ge.build()
  from uisrnn_b200 import native
  lib = native.load_library()
  ip = ctypes.POINTER(ctypes.c_int32)
  assert lib.uis_predict_bounded.argtypes == lib.uis_predict.argtypes + [ip, ip, ip]
  assert lib.uis_predict_device_bounded.argtypes == lib.uis_predict_device.argtypes + [ip, ip, ctypes.c_void_p]
  header = open(os.path.join(ROOT, 'include', 'uisrnn_b200.h')).read()
  for name, last in (('uis_predict_bounded', 'int32_t* speakers_out'),
                     ('uis_predict_device_bounded', 'int32_t* speakers_dev')):
    decl = header[header.index('int ' + name + '('):]
    decl = decl[:decl.index(';')]
    assert decl.rstrip(')').endswith(last), decl
    assert 'const int32_t* max_speakers, const int32_t* min_speakers' in decl

