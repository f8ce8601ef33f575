"""N-best predict() on the GPU: every traced golden of the reference (tests/golden small, depth-2, toy and
speaker-bounds cases) through every kernel variant that serves its shape, the (1024, 512) kernels, the device entry
point, pageable staging, decode-in-groups, a mixed bounded batch, k = beam_size = 128 and parallel_predict.

Within one call, each variant must give: plane 0 = the labels of the same call without n_best; scores = the
final_scores tap; every plane = the back-track of the kernel's own traced winners from its rank.  Against the
reference, the hypotheses match its final ranks up to one-ulp ties (test_nbest_cpu.check_nbest)."""
import ctypes

import numpy as np
import pytest

from beam_replay import backtrack
from helpers import inference_args, load_weights, uisrnn_from_weights
from test_beam_replay_cpu import GOLDEN_CASES
from test_gpu_large_models import _cached, utterances
from test_nbest_cpu import check_nbest, expected_from_trace

pytestmark = pytest.mark.gpu

LA1 = {'ffma1': dict(engine=1, lanes=1, cluster=-1), 'ffma2': dict(engine=1, lanes=2, cluster=-1)}
LA1_TOY = {'tc': dict(engine=2, lanes=6), 'cluster2': dict(engine=1, cluster=2), 'cluster4': dict(engine=1, cluster=4),
           'stat': dict(cluster=32)}


def variants(case):
  if case['look_ahead'] > 1:
    return ['tree', 'spill']
  return list(LA1) + (list(LA1_TOY) if case['model'] == 'model_toy100.npz' else [])


PARAMS = [(c, v) for c in GOLDEN_CASES for v in variants(c)]


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


def own_ranks(dbg, n_frames, test_iteration, min_speakers, k):
  """Final ranks the N-best rule picks from the kernel's own trace, and their cluster counts."""
  from uisrnn_b200.beam_cpu import nbest_ranks
  win, off = dbg['win'], dbg['off']
  finals = int(off[-1] - off[-2]) if len(off) > 1 else 0
  clusters = [max(backtrack(win, off, n_frames * test_iteration, r)) + 1 for r in range(finals)]
  return nbest_ranks(clusters, min_speakers, k), clusters


def check_call(model, x, k, kw, min_speakers=0):
  """One traced N-best call against the same call without n_best and against its own trace; returns the result."""
  plain, dbg0 = model.predict([x], trace_utt=0, **kw)
  (labels, scores, speakers, count), dbg = model.predict([x], trace_utt=0, n_best=k, **kw)
  assert np.array_equal(dbg['win'], dbg0['win']) and np.array_equal(dbg['score'], dbg0['score'])
  assert np.array_equal(labels[0][0], plain[0])
  ranks, clusters = own_ranks(dbg, len(x), kw['test_iteration'], min_speakers, k)
  c = int(count[0])
  assert c == len(ranks)
  for j, r in enumerate(ranks):
    assert labels[0][j].tolist() == backtrack(dbg['win'], dbg['off'], len(x), r)
    assert scores[0][j].view(np.int32) == dbg['final_scores'][0][r].view(np.int32)
    assert speakers[0][j] == clusters[r]
  assert (labels[0][c:] == -1).all() and np.isinf(scores[0][c:]).all() and (speakers[0][c:] == 0).all()
  return labels[0], scores[0], speakers[0], c


@pytest.mark.parametrize('case,variant', PARAMS, ids=['%s-%s' % (c['name'], v) for c, v in PARAMS])
def test_golden_case_through_kernel_variant(native, monkeypatch, case, variant):
  model = native_model(native, case['model'])
  if variant == 'spill':
    monkeypatch.setenv('UISRNN_B200_TREE_SPILL', 'force')
  opts = dict(LA1, **LA1_TOY).get(variant, {})
  mn = int(case.get('min_speakers', 0))
  kw = dict(beam_size=case['beam_size'], look_ahead=case['look_ahead'], test_iteration=case['test_iteration'],
            max_speakers=int(case.get('max_speakers', 0)), min_speakers=mn, **opts)
  for k in sorted({min(3, case['beam_size']), case['beam_size']}):
    labels, scores, _, c = check_call(model, case['x'], k, kw, mn)
    st = model.stats()
    if variant == 'tc':
      assert st['engine'] == 2
    if variant.startswith('cluster'):
      assert st['cluster'] == int(variant[-1])
    if variant == 'stat':
      assert st['cluster'] == 32
    ranks, rank_labels, final_scores, clusters = expected_from_trace(case, k)
    check_nbest(([l.tolist() for l in labels[:c]], [float(v) for v in scores[:c]], [0] * c), ranks, rank_labels,
                final_scores, [0] * len(final_scores))


@pytest.mark.parametrize('depth,look_ahead', [(1, 1), (2, 1), (1, 2)])
def test_1024x512(native, depth, look_ahead):
  _, model, _ = _cached(native, 1024, 512, depth)
  x = utterances(512, 900 + depth, (26,))[0]
  kw = dict(beam_size=5, look_ahead=look_ahead, test_iteration=1, kcap=32 if look_ahead == 1 else 16)
  assert check_call(model, x, 5, kw)[3] >= 2


def toy_batch():
  from uisrnn_b200.synth import synth_utt
  return [synth_utt(9100 + u, n_frames=40 + 9 * u, n_spk=4, noise=0.06)[0] for u in range(10)] + \
      [np.zeros((0, 256))]


def test_batch_paths_agree_with_single_calls(native, monkeypatch):
  """Device entry, pageable staging, decode in groups, and per-utterance bounds give what single calls give."""
  import torch
  model = native_model(native, 'model_toy100.npz')
  xs, k = toy_batch(), 4
  mx = np.array([2, 0, 3, 0, 2, 4, 0, 1, 0, 3, 0], np.int32)
  mn = np.array([0, 0, 2, 3, 0, 0, 0, 1, 2, 0, 0], np.int32)
  single = [model.predict([x], n_best=k, max_speakers=int(a), min_speakers=int(b)) for x, a, b in zip(xs, mx, mn)]
  plain = model.predict(xs, max_speakers=mx, min_speakers=mn)

  def same(out):
    labels, scores, speakers, count = out
    for u, (lab, sc, sp, c) in enumerate(single):
      # (a single utterance runs a latency-mode kernel: same search, scores equal to rounding)
      assert np.array_equal(labels[u], lab[0]) and np.allclose(scores[u], sc[0], rtol=1e-5, atol=0), u
      assert np.array_equal(speakers[u], sp[0]) and count[u] == c[0], u
      assert np.array_equal(labels[u][0], plain[u])
  same(model.predict(xs, n_best=k, max_speakers=mx, min_speakers=mn))
  assert model.stats()['groups'] == 1
  monkeypatch.setenv('UISRNN_B200_MAX_ROWS', '150')
  same(model.predict(xs, n_best=k, max_speakers=mx, min_speakers=mn))
  assert model.stats()['groups'] > 1
  monkeypatch.delenv('UISRNN_B200_MAX_ROWS')
  monkeypatch.setenv('UISRNN_B200_HOST_STAGING', '1')
  same(model.predict(xs, n_best=k, max_speakers=mx, min_speakers=mn))
  assert model.stats()['staged'] == 1
  monkeypatch.delenv('UISRNN_B200_HOST_STAGING')
  # device entry: plane-major labels [k][rows]
  off = np.zeros(len(xs) + 1, np.int64)
  np.cumsum([len(x) for x in xs], out=off[1:])
  x = torch.from_numpy(np.concatenate(xs).astype(np.float32)).cuda()
  lab = torch.full((k, int(off[-1])), -7, dtype=torch.int32, device='cuda')
  sc = torch.zeros((len(xs), k), dtype=torch.float32, device='cuda')
  sp = torch.zeros((len(xs), k), dtype=torch.int32, device='cuda')
  cnt = torch.zeros(len(xs), dtype=torch.int32, device='cuda')
  model.predict_device(x.data_ptr(), off, lab.data_ptr(), max_speakers=mx, min_speakers=mn, n_best=k,
                       scores_ptr=sc.data_ptr(), nbest_speakers_ptr=sp.data_ptr(), count_ptr=cnt.data_ptr())
  torch.cuda.synchronize()
  lab = lab.cpu().numpy()
  same(([lab[:, off[u]:off[u + 1]] for u in range(len(xs))], sc.cpu().numpy(), sp.cpu().numpy(), cnt.cpu().numpy()))
  assert single[-1][3][0] == 0  # the empty utterance returns no hypothesis


def test_beam_128_all_ranks(native):
  model = native_model(native, 'model_toy100.npz')
  from uisrnn_b200.synth import synth_utt
  x = synth_utt(9300, n_frames=70, n_spk=4, noise=0.06)[0]
  # (beam 128 shrinks the default kcap to what shared memory holds; max_speakers 4 keeps K below it)
  kw = dict(beam_size=128, look_ahead=1, test_iteration=2, engine=1, lanes=1, cluster=-1, max_speakers=4)
  assert check_call(model, x, 128, kw)[3] == 128


def test_validation(native):
  model = native_model(native, 'model_small.npz')
  x = np.zeros((5, 64))
  for bad in (0, 11, -1, 2.5, True):
    with pytest.raises(ValueError):
      model.predict([x], beam_size=10, n_best=bad)
  lib = native.load_library()
  opts = model._opts(10, 1, 2, 0, 0)  # pylint: disable=protected-access
  off = np.zeros(1, np.int64)
  for k in (0, 11):
    rc = lib.uis_predict_device_nbest(model._h, None, off.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), 0,  # pylint: disable=protected-access
                                      ctypes.byref(opts), None, None, None, None, k, ctypes.byref(native.NBestOut()))
    assert rc == native.UIS_ERR_INVALID


def test_uisrnn_and_parallel_predict(native):
  import torch
  from uisrnn_b200.uisrnn import NBest, parallel_predict
  model = uisrnn_from_weights(load_weights('model_toy100.npz'), enable_cuda=True)
  args = inference_args(10, 1, 2)
  xs = toy_batch()[:4]
  out = model.predict(xs, args, n_best=3, max_speakers=3)
  assert all(isinstance(o, NBest) for o in out)
  assert [o.labels[0] for o in out] == model.predict(xs, args, max_speakers=3)
  assert model.predict(xs[0], args, n_best=3) == model.predict([xs[0]], args, n_best=3)[0]
  if torch.cuda.device_count() < 2:
    pytest.skip('parallel_predict over devices needs two GPUs')
  assert parallel_predict(model, xs, args, num_processes=2, n_best=3, max_speakers=3) == out
