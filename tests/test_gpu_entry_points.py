"""The plain C entry points that NativeModel no longer calls -- uis_predict, uis_predict_bounded, uis_predict_nbest,
their device forms, uis_score and uis_score_device -- called directly through ctypes.  Each must give, bit for bit,
what the NativeModel call gives (a one-pair sweep of the model's own pair): labels, cluster counts, N-best scores
and per-frame score increments.  Also: the model's own log tables are picked by value, so plain calls and sweeps can
alternate on one handle without changing a result."""
import ctypes

import numpy as np
import pytest

from helpers import load_weights
from test_beam_replay_cpu import GOLDEN_CASES
from test_gpu_large_models import large_model, utterances
from test_gpu_nbest import LA1, LA1_TOY, variants

pytestmark = pytest.mark.gpu

CASES = {c['name']: c for c in GOLDEN_CASES}
VP = ctypes.c_void_p
IP = ctypes.POINTER(ctypes.c_int32)
FP = ctypes.POINTER(ctypes.c_float)
LP = ctypes.POINTER(ctypes.c_int64)


@pytest.fixture(scope='module')
def native():
  from uisrnn_b200 import native as nat
  nat.load_library()
  return nat


_MODELS = {}


def model_for(native, name, weights=None):
  if name not in _MODELS:
    _MODELS[name] = native.NativeModel(weights if weights is not None else load_weights(name))
  return _MODELS[name]


def batch(x):
  """One utterance, a prefix of it and an empty one."""
  return [x, x[:len(x) // 2 + 1], np.zeros((0, x.shape[1]))]


def ptr(a):
  return a.ctypes.data_as(IP) if a is not None else None


def opts_of(model, kw):
  return model._opts(kw['beam_size'], kw['look_ahead'], kw['test_iteration'], kw.get('kcap', 0), 0,  # pylint: disable=protected-access
                     kw.get('lanes', 0), kw.get('cluster', 0), kw.get('engine', 0))


def host_call(native, model, xs, kw, mx=None, mn=None, k=None):
  """uis_predict (no bounds, no k), uis_predict_bounded (bounds; speakers_out) or uis_predict_nbest (k) on host
  buffers.  Returns (labels [U][planes][N_u], speakers [U] or None, scores [U][k], N-best speakers [U][k], count [U])."""
  lib = native.load_library()
  xs = [np.ascontiguousarray(x, np.float64) for x in xs]
  n = len(xs)
  lens = np.array([len(x) for x in xs] or [0], np.int64)
  outs = [np.full((k or 1, len(x)), -7, np.int32) for x in xs]
  ins, labs = (VP * max(n, 1))(*[x.ctypes.data for x in xs]), (VP * max(n, 1))(*[o.ctypes.data for o in outs])
  opts = opts_of(model, kw)
  if k is not None:
    scores, spk, count = np.zeros((n, k), np.float32), np.zeros((n, k), np.int32), np.zeros(n, np.int32)
    nb = native.NBestOut(labs, None, scores.ctypes.data_as(FP), ptr(spk), ptr(count))
    rc = lib.uis_predict_nbest(model._h, ins, lens.ctypes.data_as(LP), n, ctypes.byref(opts), None, None, ptr(mx),  # pylint: disable=protected-access
                               ptr(mn), k, ctypes.byref(nb))
    assert rc == 0, lib.uis_last_error()
    return outs, None, scores, spk, count
  if mx is None and mn is None:
    rc = lib.uis_predict(model._h, ins, lens.ctypes.data_as(LP), n, ctypes.byref(opts), labs, None, None)  # pylint: disable=protected-access
    assert rc == 0, lib.uis_last_error()
    return outs, None, None, None, None
  spk = np.full(max(n, 1), -7, np.int32)
  rc = lib.uis_predict_bounded(model._h, ins, lens.ctypes.data_as(LP), n, ctypes.byref(opts), labs, None, None,  # pylint: disable=protected-access
                               ptr(mx), ptr(mn), ptr(spk))
  assert rc == 0, lib.uis_last_error()
  return outs, spk[:n], None, None, None


def device_rows(xs):
  import torch
  off = np.zeros(len(xs) + 1, np.int64)
  np.cumsum([len(x) for x in xs], out=off[1:])
  return torch.from_numpy(np.concatenate(xs).astype(np.float32)).cuda(), off


def device_call(native, model, xs, kw, mx=None, mn=None, k=None, routed=False):
  """uis_predict_device / uis_predict_device_bounded / uis_predict_device_nbest, or with routed=True the NativeModel
  call (predict_device(n_best=k or 1), a one-pair sweep).  Returns (labels [planes][rows], scores, N-best speakers,
  count, speakers_dev) as numpy arrays (None where the entry has no such output)."""
  import torch
  lib = native.load_library()
  x, off = device_rows(xs)
  n, rows, planes = len(xs), int(off[-1]), k or 1
  lab = torch.full((planes, max(rows, 1)), -7, dtype=torch.int32, device='cuda')
  sc = torch.zeros((n, planes), dtype=torch.float32, device='cuda')
  sp = torch.zeros((n, planes), dtype=torch.int32, device='cuda')
  cnt = torch.zeros(n, dtype=torch.int32, device='cuda')
  spk = torch.full((n,), -7, dtype=torch.int32, device='cuda')
  opts = opts_of(model, kw)
  offp = off.ctypes.data_as(LP)
  got_nbest = routed or k is not None
  if routed:
    model.predict_device(x.data_ptr(), off, lab.data_ptr(), beam_size=kw['beam_size'], look_ahead=kw['look_ahead'],
                         test_iteration=kw['test_iteration'], kcap=kw.get('kcap', 0), lanes=kw.get('lanes', 0),
                         cluster=kw.get('cluster', 0), engine=kw.get('engine', 0), max_speakers=mx, min_speakers=mn,
                         n_best=planes, scores_ptr=sc.data_ptr(), nbest_speakers_ptr=sp.data_ptr(),
                         count_ptr=cnt.data_ptr())
  elif k is not None:
    nb = native.NBestOut(None, VP(lab.data_ptr()), ctypes.cast(VP(sc.data_ptr()), FP), ctypes.cast(VP(sp.data_ptr()), IP),
                         ctypes.cast(VP(cnt.data_ptr()), IP))
    rc = lib.uis_predict_device_nbest(model._h, VP(x.data_ptr()), offp, n, ctypes.byref(opts), None, None, ptr(mx),  # pylint: disable=protected-access
                                      ptr(mn), k, ctypes.byref(nb))
    assert rc == 0, lib.uis_last_error()
  elif mx is None and mn is None:
    rc = lib.uis_predict_device(model._h, VP(x.data_ptr()), offp, n, ctypes.byref(opts), VP(lab.data_ptr()), None, None)  # pylint: disable=protected-access
    assert rc == 0, lib.uis_last_error()
  else:
    rc = lib.uis_predict_device_bounded(model._h, VP(x.data_ptr()), offp, n, ctypes.byref(opts), VP(lab.data_ptr()),  # pylint: disable=protected-access
                                        None, None, ptr(mx), ptr(mn), VP(spk.data_ptr()))
    assert rc == 0, lib.uis_last_error()
  torch.cuda.synchronize()
  lab = lab.cpu().numpy()[:, :rows]
  if got_nbest:
    return lab, sc.cpu().numpy(), sp.cpu().numpy(), cnt.cpu().numpy(), None
  return lab, None, None, None, spk.cpu().numpy()


def same_bits(a, b):
  a, b = np.asarray(a), np.asarray(b)
  return a.shape == b.shape and np.array_equal(a.view(np.int32) if a.dtype == np.float32 else a,
                                               b.view(np.int32) if b.dtype == np.float32 else b)


def check_predict(native, model, xs, kw, mx, mn, k):
  """Every legacy predict entry against the NativeModel call with the same arguments."""
  off = np.zeros(len(xs) + 1, np.int64)
  np.cumsum([len(x) for x in xs], out=off[1:])
  plain = model.predict(xs, **kw)
  bounded, speakers = model.predict(xs, max_speakers=mx, min_speakers=mn, return_speakers=True, **kw)
  labels, scores, nb_spk, count = model.predict(xs, max_speakers=mx, min_speakers=mn, n_best=k, **kw)
  # host entries
  got = host_call(native, model, xs, kw)[0]
  assert all(same_bits(g[0], p) for g, p in zip(got, plain))
  got, spk = host_call(native, model, xs, kw, mx, mn)[:2]
  assert all(same_bits(g[0], b) for g, b in zip(got, bounded)) and same_bits(spk, speakers)
  got, _, sc, sp, cnt = host_call(native, model, xs, kw, mx, mn, k)
  assert all(same_bits(g, l) for g, l in zip(got, labels))
  assert same_bits(sc, scores) and same_bits(sp, nb_spk) and same_bits(cnt, count)
  # device entries, against the device call NativeModel routes through the sweep entry
  lab1, _, sp1, _, _ = device_call(native, model, xs, kw, routed=True)
  assert same_bits(device_call(native, model, xs, kw)[0], lab1)
  assert same_bits(lab1[0], np.concatenate(plain))
  lab1, _, sp1, _, _ = device_call(native, model, xs, kw, mx, mn, routed=True)
  lab, _, _, _, spk = device_call(native, model, xs, kw, mx, mn)
  assert same_bits(lab, lab1) and same_bits(spk, sp1[:, 0]) and same_bits(spk, speakers)
  routed = device_call(native, model, xs, kw, mx, mn, k, routed=True)
  legacy = device_call(native, model, xs, kw, mx, mn, k)
  assert all(same_bits(a, b) for a, b in zip(legacy[:4], routed[:4]))
  assert same_bits(routed[0], np.concatenate(labels, axis=1))
  check_score(native, model, xs, plain)


def check_score(native, model, xs, decoded):
  """uis_score / uis_score_device (per-frame increments) against NativeModel.score / score_device on the
  canonical form of the decoded labels."""
  import torch
  from uisrnn_b200.uisrnn import canonical_labels
  lib = native.load_library()
  labs = [canonical_labels(l) for l in decoded]
  totals, frames = model.score(xs, labs, per_frame=True)
  keep = [np.ascontiguousarray(x, np.float64) for x in xs]
  n = len(xs)
  lens = np.array([len(x) for x in xs], np.int64)
  scores = np.full(n, np.nan, np.float32)
  inc = [np.full(len(x), np.nan, np.float32) for x in xs]
  arr = lambda a: (VP * n)(*[v.ctypes.data for v in a])
  rc = lib.uis_score(model._h, arr(keep), lens.ctypes.data_as(LP), n, arr(labs), scores.ctypes.data_as(FP), arr(inc),  # pylint: disable=protected-access
                     None)
  assert rc == 0, lib.uis_last_error()
  assert same_bits(scores, totals) and all(same_bits(a, b) for a, b in zip(inc, frames))
  x, off = device_rows(xs)
  lab = torch.from_numpy(np.concatenate(labs)).cuda()
  outs = []
  for legacy in (True, False):
    sc = torch.full((n,), float('nan'), dtype=torch.float32, device='cuda')
    fr = torch.full((max(int(off[-1]), 1),), float('nan'), dtype=torch.float32, device='cuda')
    if legacy:
      rc = lib.uis_score_device(model._h, VP(x.data_ptr()), off.ctypes.data_as(LP), n, VP(lab.data_ptr()),  # pylint: disable=protected-access
                                VP(sc.data_ptr()), VP(fr.data_ptr()), None)
      assert rc == 0, lib.uis_last_error()
    else:
      model.score_device(x.data_ptr(), off, lab.data_ptr(), sc.data_ptr(), frame_ptr=fr.data_ptr())
    torch.cuda.synchronize()
    outs.append((sc.cpu().numpy(), fr.cpu().numpy()[:int(off[-1])]))
  assert same_bits(outs[0][0], outs[1][0]) and same_bits(outs[0][1], outs[1][1])
  assert same_bits(outs[0][1], np.concatenate(frames))


GOLDEN = [(name, v) for name in ('toy_u0', 'la2b') for v in variants(CASES[name])]


@pytest.mark.parametrize('name,variant', GOLDEN, ids=['%s-%s' % g for g in GOLDEN])
def test_legacy_entries_match_routed_calls(native, monkeypatch, name, variant):
  case = CASES[name]
  if variant == 'spill':
    monkeypatch.setenv('UISRNN_B200_TREE_SPILL', 'force')
  model = model_for(native, case['model'])
  kw = dict(beam_size=case['beam_size'], look_ahead=case['look_ahead'], test_iteration=case['test_iteration'],
            **dict(LA1, **LA1_TOY).get(variant, {}))
  mx, mn = np.array([0, 3, 0], np.int32), np.array([2, 0, 0], np.int32)
  check_predict(native, model, batch(case['x']), kw, mx, mn, min(3, case['beam_size']))


@pytest.mark.parametrize('which', ['depth2', 'zero_padded'])
def test_legacy_entries_other_shapes(native, which):
  from uisrnn_b200.synth import synth_utt
  if which == 'depth2':
    model = model_for(native, 'model_small_d2.npz')
    x = synth_utt(9700, n_frames=57, dim=64, n_spk=3, noise=0.05)[0]
  else:  # hidden 100 / dim 48 runs zero-padded in the (128, 64) kernels
    model = model_for(native, 'padded_100x48', large_model(100, 48, 1, seed=148))
    x = utterances(48, 9700, (57,))[0]
  kw = dict(beam_size=8, look_ahead=1, test_iteration=2, kcap=64)  # (room for every cluster these decodes open)
  check_predict(native, model, batch(x), kw, np.array([3, 0, 2], np.int32), np.array([2, 0, 0], np.int32), 4)


def test_own_log_tables_by_value(native):
  """plain -> sweep of other pairs -> plain -> sweep holding the model's pair, on one handle: every result is what a
  fresh handle's plain call gives for that pair."""
  from uisrnn_b200.synth import synth_utt
  w = load_weights('model_small.npz')
  own = (float(w['crp_alpha']), float(w['transition_bias']))
  others = [(0.5, 0.2), (2.0, 0.05)]
  xs = [synth_utt(9800 + u, n_frames=40 + 7 * u, dim=64, n_spk=3, noise=0.06)[0] for u in range(4)]
  kw = dict(beam_size=10, look_ahead=1, test_iteration=2, n_best=3)

  def fresh(pair):
    return native.NativeModel(dict(w, crp_alpha=pair[0], transition_bias=pair[1])).predict(xs, **kw)

  want = {pair: fresh(pair) for pair in [own] + others}

  def same(got, pair):
    labels, scores, speakers, count = got
    w_labels, w_scores, w_speakers, w_count = want[pair]
    assert all(same_bits(a, b) for a, b in zip(labels, w_labels)), pair
    assert same_bits(scores, w_scores) and same_bits(speakers, w_speakers) and same_bits(count, w_count), pair

  def same_sweep(got, pairs):
    labels, scores, speakers, count = got
    for c, pair in enumerate(pairs):
      same(([l[c] for l in labels], scores[c], speakers[c], count[c]), pair)

  model = native.NativeModel(w)
  same(model.predict(xs, **kw), own)
  same_sweep(model.predict_sweep(xs, others, **kw), others)
  same(model.predict(xs, **kw), own)
  lab, _, sc, sp, cnt = host_call(native, model, xs, kw, k=3)
  same((lab, sc, sp, cnt), own)
  mixed = [others[0], own, others[1]]
  same_sweep(model.predict_sweep(xs, mixed, **kw), mixed)
  same(model.predict(xs, **kw), own)
