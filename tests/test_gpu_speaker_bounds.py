"""Speaker bounds on the GPU: every case of tests/golden/speaker_bounds_cases.npz (the reference's own search with the
bounds applied) through every kernel variant that serves its shape, the (1024, 512) kernels against the bounded CPU
oracle, non-binding bounds against the unbounded goldens, a mixed batch, the min-bound fallback, the device entry
point and the public paths."""
import os
import socket
import sys
import warnings

import numpy as np
import pytest

from helpers import ROOT, compare_trace, inference_args, load_weights, oracle_model, toy_utterances, \
    uisrnn_from_weights
import speaker_bounds_oracle as SB
from test_gpu_large_models import _cached, utterances
from test_speaker_bounds_cpu import CASES

pytestmark = pytest.mark.gpu

LA1 = {'ffma1': dict(engine=1, lanes=1, cluster=-1), 'ffma2': dict(engine=1, lanes=2, cluster=-1)}
LA1_TOY = {'tc': dict(engine=2), 'cluster2': dict(engine=1, cluster=2), 'cluster4': dict(engine=1, cluster=4),
           'stat': dict(cluster=32)}


def variants(case):
  if case['look_ahead'] > 1:
    return ['tree', 'spill']
  return list(LA1) + (list(LA1_TOY) if case['model'] == 'model_toy100.npz' else [])


PARAMS = [(c, v) for c in CASES for v in variants(c)]


@pytest.fixture(scope='module')
def native():
  from uisrnn_b200 import native as nat
  nat.load_library()
  return nat


_MODELS = {}


def native_model(native, name):
  if name not in _MODELS:
    _MODELS[name] = native.NativeModel(load_weights(name))
  return _MODELS[name]


def bound_kw(case):
  return dict(beam_size=case['beam_size'], look_ahead=case['look_ahead'], test_iteration=case['test_iteration'],
              max_speakers=case['max_speakers'], min_speakers=case['min_speakers'])


@pytest.mark.parametrize('case,variant', PARAMS, ids=['%s-%s' % (c['name'], v) for c, v in PARAMS])
def test_fixture_case_through_kernel_variant(native, monkeypatch, case, variant):
  model = native_model(native, case['model'])
  if variant == 'spill':
    monkeypatch.setenv('UISRNN_B200_TREE_SPILL', 'force')
  opts = dict(LA1, **LA1_TOY).get(variant, {})
  kw = dict(bound_kw(case), return_speakers=True, **opts)
  (labels, speakers), dbg = model.predict([case['x']], trace_utt=0, **kw)  # traced in every variant
  compare_trace(dbg['win'], dbg['score'], dbg['off'], case['win'], case['score'], case['off'])
  st = model.stats()
  if variant == 'tc':
    assert st['engine'] == 2
  if variant.startswith('cluster'):
    assert st['cluster'] == int(variant[-1])
  if variant == 'stat':
    assert st['cluster'] == 32
  assert labels[0].tolist() == case['labels'].tolist()
  assert speakers[0] == case['final_k'][int(case['chosen'])]


@pytest.mark.parametrize('depth,look_ahead', [(1, 1), (2, 1), (1, 3), (2, 3)])
def test_1024x512_against_bounded_oracle(native, depth, look_ahead):
  _, model, om = _cached(native, 1024, 512, depth)
  xs = utterances(512, 800 + depth, (24, 17))
  beam, titer = 5, 1
  free = [max(uis_labels) + 1 for uis_labels in
          (SB.predict_single(om, x, beam, look_ahead, titer) for x in xs)]
  bounds = [max(1, k - 1) for k in free]
  assert max(free) > 2  # the bound binds somewhere
  got, speakers = model.predict(xs, beam_size=beam, look_ahead=look_ahead, test_iteration=titer,
                                max_speakers=bounds, return_speakers=True)
  for x, g, k, mx in zip(xs, got, speakers, bounds):
    rec = {}
    want = SB.predict_single(om, x, beam, look_ahead, titer, max_speakers=mx, record=rec)
    assert g.tolist() == want and k == rec['final_k'][0] and g.max() < mx


def test_non_binding_bounds_match_the_unbounded_goldens(native):
  model = native_model(native, 'model_toy100.npz')
  xs, labs = toy_utterances()
  got = model.predict(xs, max_speakers=64, min_speakers=1, kcap=64)
  assert [g.tolist() for g in got] == [l.tolist() for l in labs]
  from uisrnn_b200.synth import synth_utt
  g = np.load(os.path.join(ROOT, 'tests', 'golden', 'synth500.npz'))
  xs = [synth_utt(int(s))[0] for s in g['seeds']]
  got = model.predict(xs, max_speakers=[64, 40], min_speakers=[1, 0], kcap=64)
  assert [r.tolist() for r in got] == [l.tolist() for l in g['labels']]


def mixed_batch():
  from uisrnn_b200.synth import synth_utt
  xs = [synth_utt(9000 + u, n_frames=60 + 7 * u, n_spk=5, noise=0.059)[0] for u in range(12)]
  mx = np.array([2, 0, 3, 1, 0, 2, 4, 0, 2, 3, 0, 1], np.int32)
  mn = np.array([0, 0, 2, 1, 3, 0, 0, 0, 2, 0, 0, 0], np.int32)
  return xs, mx, mn


def test_mixed_batch(native):
  model = native_model(native, 'model_toy100.npz')
  xs, mx, mn = mixed_batch()
  ref, spk = model.predict(xs, max_speakers=mx, min_speakers=mn, return_speakers=True)
  plain = model.predict(xs)
  for u in range(len(xs)):
    if mx[u] == 0 and mn[u] == 0:
      assert ref[u].tolist() == plain[u].tolist()
    if mx[u]:
      assert ref[u].max() < mx[u] and spk[u] <= mx[u]
  perm = np.random.default_rng(3).permutation(len(xs))
  for kw in (dict(n_ctas=1), dict(n_ctas=3, lanes=2), dict(engine=1), dict(engine=2)):
    got, s2 = model.predict([xs[i] for i in perm], max_speakers=mx[perm], min_speakers=mn[perm],
                            return_speakers=True, **kw)
    for j, i in enumerate(perm):
      assert got[j].tolist() == ref[i].tolist() and s2[j] == spk[i], (kw, i)


def test_min_bound_fallback_warns(native):
  case = {c['name']: c for c in CASES}['s_min_fallback']
  model = native_model(native, case['model'])
  labels, spk = model.predict([case['x']], return_speakers=True, **bound_kw(case))
  assert labels[0].tolist() == case['final_traces'][0].tolist() and spk[0] < case['min_speakers']
  um = uisrnn_from_weights(load_weights(case['model']), enable_cuda=True)
  args = inference_args(case['beam_size'], case['look_ahead'], case['test_iteration'])
  with warnings.catch_warnings(record=True) as caught:
    warnings.simplefilter('always')
    out = um.predict([case['x'][:3], case['x']], args, min_speakers=[0, case['min_speakers']])
  assert out[1] == case['labels'].tolist()
  assert len([w for w in caught if 'min_speakers' in str(w.message) and '[1]' in str(w.message)]) == 1


def test_device_entry_point(native):
  import torch
  model = native_model(native, 'model_toy100.npz')
  xs, mx, mn = mixed_batch()
  want, spk = model.predict(xs, max_speakers=mx, min_speakers=mn, return_speakers=True)
  x = torch.from_numpy(np.concatenate(xs).astype(np.float32)).cuda()
  off = np.concatenate([[0], np.cumsum([len(v) for v in xs])]).astype(np.int64)
  lab = torch.empty(int(off[-1]), dtype=torch.int32, device='cuda')
  dspk = torch.full((len(xs),), -7, dtype=torch.int32, device='cuda')
  model.predict_device(x.data_ptr(), off, lab.data_ptr(), max_speakers=mx, min_speakers=mn,
                       speakers_ptr=dspk.data_ptr())
  torch.cuda.synchronize()
  assert np.array_equal(lab.cpu().numpy(), np.concatenate(want))
  assert np.array_equal(dspk.cpu().numpy(), spk)


def test_public_paths(native, monkeypatch):
  from uisrnn_b200.uisrnn import parallel_predict
  case = {c['name']: c for c in CASES}['toy_b10_la1_t2']
  um = uisrnn_from_weights(load_weights('model_toy100.npz'), enable_cuda=True)
  args = inference_args(case['beam_size'], case['look_ahead'], case['test_iteration'])
  assert um.predict(case['x'], args, max_speakers=case['max_speakers']) == case['labels'].tolist()
  assert um.predict_single(case['x'], args, max_speakers=case['max_speakers']) == case['labels'].tolist()
  xs, mx, mn = mixed_batch()
  want = [w.tolist() for w in native_model(native, 'model_toy100.npz').predict(xs, max_speakers=mx, min_speakers=mn)]
  with warnings.catch_warnings():
    warnings.simplefilter('ignore')
    assert um.predict(xs, inference_args(), max_speakers=mx, min_speakers=mn) == want
    assert parallel_predict(um, xs, inference_args(), max_speakers=mx, min_speakers=mn) == want
    monkeypatch.setenv('UISRNN_B200_MAX_ROWS', '150')  # decoded in groups: the bounds follow their utterances
    assert um.predict(xs, inference_args(), max_speakers=mx, min_speakers=mn) == want


def _sharded_worker(rank, world, port, out_dir):
  sys.path.insert(0, ROOT)
  sys.path.insert(0, os.path.join(ROOT, 'tests'))
  import warnings as w
  import torch.distributed as dist
  from uisrnn_b200.distributed import predict_sharded
  w.simplefilter('ignore')
  dist.init_process_group('gloo', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=world)
  um = uisrnn_from_weights(load_weights('model_toy100.npz'), enable_cuda=True)
  xs, mx, mn = mixed_batch()
  got = predict_sharded(um, xs, inference_args(), max_speakers=mx, min_speakers=mn)
  np.save(os.path.join(out_dir, 'rank%d.npy' % rank), np.array(got, dtype=object), allow_pickle=True)
  dist.destroy_process_group()


def test_predict_sharded_gloo_world2(native, tmp_path):
  import torch.multiprocessing as mp
  with socket.socket() as s:
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
  mp.spawn(_sharded_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
  xs, mx, mn = mixed_batch()
  want = [w.tolist() for w in native_model(native, 'model_toy100.npz').predict(xs, max_speakers=mx, min_speakers=mn)]
  for rank in (0, 1):
    got = np.load(str(tmp_path / ('rank%d.npy' % rank)), allow_pickle=True).tolist()
    assert [list(g) for g in got] == want
