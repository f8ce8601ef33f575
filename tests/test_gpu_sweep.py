"""Decoding-parameter sweeps on the GPU: one call under C (crp_alpha, transition_bias) pairs against C plain calls on
models created with those pairs, under the same forced kernel (tensor cores, FFMA with 1 and 2 lanes, cluster mode,
stationary weights, the look-ahead tree kernel in shared memory and through the spill arena, depth 2, the (1024, 512)
kernels, a zero-padded shape, beam 64).  Results do not depend on how a call is composed within one engine, so every
label, N-best score, speaker count and hypothesis count must be bit-identical.  Also: the oracle's labels per pair,
speaker bounds with n_best, decode-in-groups, the device entry point on a side stream, traced jobs, score sweeps
(totals and per-frame increments, long logtot tables, the chain kernel run once) and the C ABI's argument checks."""
import ctypes

import numpy as np
import pytest

import beam_replay as R
from helpers import load_weights, toy_utterances, uis_oracle
from test_gpu_large_models import utterances
from test_gpu_score_frames import rescore
from test_gpu_step_replay import random_weights
from test_sweep_cpu import sweep_golden

pytestmark = pytest.mark.gpu

# the model's own pair of the small / toy fixtures is added per model; these are far apart (distinct labels per pair)
PAIRS = [(1e-3, 0.5), (30.0, 0.01), (0.2, 0.9)]


@pytest.fixture(scope='module')
def native():
  from uisrnn_b200 import native as nat
  nat.load_library()
  return nat


def with_pair(w, pair):
  w = dict(w)
  w['crp_alpha'], w['transition_bias'] = pair
  return w


def own_pair(w):
  return (float(w['crp_alpha']), float(w['transition_bias']))


_PLAIN = {}


def plain_model(native, key, w, pair):
  if (key, pair) not in _PLAIN:
    _PLAIN[(key, pair)] = native.NativeModel(with_pair(w, pair))
  return _PLAIN[(key, pair)]


def check_sweep(native, key, w, xs, pairs, n_best=3, **kw):
  """Sweep on a model built from `w` against plain N-best calls on one model per pair; returns the sweep's labels."""
  sweep_model = plain_model(native, key, w, own_pair(w))
  labels, scores, speakers, count = sweep_model.predict_sweep(xs, pairs, n_best=n_best, **kw)
  st = sweep_model.stats()
  assert st['utterances'] == len(xs) * len(pairs) and st['frames'] == sum(len(x) for x in xs)
  for c, pair in enumerate(pairs):
    lab, sc, sp, cnt = plain_model(native, key, w, pair).predict(xs, n_best=n_best, **kw)
    for u in range(len(xs)):
      assert np.array_equal(labels[u][c], lab[u]), (pair, u)
    assert np.array_equal(scores[c].view(np.uint32), sc.view(np.uint32)), pair
    assert np.array_equal(speakers[c], sp) and np.array_equal(count[c], cnt), pair
  return labels


def distinct(model, xs, pairs, labels_too=True, **kw):
  """Every pair's N-best scores differ from every other pair's (and, with labels_too, some pairs' labels differ), so
  that a config mix-up cannot pass the bit-identity checks unseen."""
  labels, scores, _, _ = model.predict_sweep(xs, pairs, n_best=3, **kw)
  for a in range(len(pairs)):
    for b in range(a + 1, len(pairs)):
      assert not np.array_equal(scores[a], scores[b]), (pairs[a], pairs[b])
  if labels_too:
    assert any(not np.array_equal(l[a][0], l[b][0]) for l in labels for a in range(len(pairs)) for b in range(a))


TOY_VARIANTS = {'tc6': dict(engine=2, lanes=6), 'ffma1': dict(engine=1, lanes=1, cluster=-1),
                'ffma2': dict(engine=1, lanes=2, cluster=-1), 'cluster4': dict(engine=1, cluster=4)}


@pytest.mark.parametrize('variant', list(TOY_VARIANTS))
def test_toy_sweep_matches_plain_calls_and_oracle(native, variant):
  w = load_weights('model_toy100.npz')
  xs, _ = toy_utterances()
  xs = [x[:48] for x in xs[:6]]
  pairs = [own_pair(w)] + PAIRS
  kw = dict(beam_size=10, look_ahead=1, test_iteration=2, **TOY_VARIANTS[variant])
  labels = check_sweep(native, 'toy', w, xs, pairs, **kw)
  distinct(plain_model(native, 'toy', w, own_pair(w)), xs, pairs, **kw)
  for c, pair in enumerate(pairs[:2]):  # the reference's search under the pair (the numpy oracle; slow at hidden 512)
    om = uis_oracle.OracleModel(with_pair(w, pair))
    for u in range(1):
      assert labels[u][c][0].tolist() == uis_oracle.predict_single(om, xs[u], beam_size=10, look_ahead=1,
                                                                   test_iteration=2)


def test_stationary_weights_one_utterance_four_pairs(native):
  w = load_weights('model_toy100.npz')
  xs = [toy_utterances()[0][0][:80]]
  kw = dict(beam_size=10, look_ahead=1, test_iteration=2, cluster=32)
  model = plain_model(native, 'toy', w, own_pair(w))
  model.predict_sweep(xs, [own_pair(w)] + PAIRS, n_best=3, **kw)
  assert model.stats()['cluster'] == 32  # the sweep itself ran the stationary-weights kernel
  check_sweep(native, 'toy', w, xs, [own_pair(w)] + PAIRS, **kw)


# ---- the reference's own decodes and losses under non-default pairs (tests/golden/sweep_cases.npz)

@pytest.mark.parametrize('variant', list(TOY_VARIANTS))
def test_toy_sweep_matches_reference_fixture(native, variant):
  fx, _, _ = sweep_golden()
  w = load_weights('model_toy100.npz')
  labels, _, _, _ = plain_model(native, 'toy', w, own_pair(w)).predict_sweep(
      fx['xs'], fx['pairs'], beam_size=10, look_ahead=1, test_iteration=2, **TOY_VARIANTS[variant])
  for c, pair in enumerate(fx['pairs']):
    for i in range(len(fx['xs'])):
      assert labels[i][c][0].tolist() == fx['labels'][c][i].tolist(), (pair, fx['utts'][i])


@pytest.mark.parametrize('spill', ['tree', 'spill'])
def test_tree_sweep_matches_reference_traces(native, monkeypatch, spill):
  if spill == 'spill':
    monkeypatch.setenv('UISRNN_B200_TREE_SPILL', 'force')
  _, fx, _ = sweep_golden()
  w = load_weights('model_small.npz')
  b, la, ti = fx['args']
  labels, scores, _, count = plain_model(native, 'small', w, own_pair(w)).predict_sweep(
      fx['xs'], fx['pairs'], n_best=b, beam_size=b, look_ahead=la, test_iteration=ti, kcap=64)
  for c, pair in enumerate(fx['pairs']):
    for i, tr in enumerate(fx['traces'][c]):
      assert labels[i][c][0].tolist() == tr['labels'].tolist(), (pair, i)
      want = tr['final_scores'][:count[c][i]]
      assert np.allclose(scores[c][i][:count[c][i]], want, rtol=1e-5, atol=0), (pair, i)


@pytest.mark.parametrize('model_name', ['model_toy100.npz', 'model_small.npz'])
def test_score_sweep_matches_reference_losses_and_rescore(native, model_name):
  """Per frame within the float64 rescore's allowance (INC_RTOL), like the reference's own losses."""
  _, _, cases = sweep_golden()
  cases = [c for c in cases if c['model'] == model_name]
  w = load_weights(model_name)
  model = plain_model(native, model_name, w, own_pair(w))
  mean0 = model.constants()[0]
  pairs = sorted({c['pair'] for c in cases})
  xs, labs = [c['x'] for c in cases], [c['labels'].astype(np.int32) for c in cases]
  tot, inc = model.score_sweep(xs, labs, pairs, per_frame=True)
  for i, case in enumerate(cases):
    c = pairs.index(case['pair'])
    f64, gauss = rescore(with_pair(w, case['pair']), [case['x']], [case['labels']], mean0)
    assert R.frame_share(inc[i][c], f64[0], gauss[0]).max() <= 1, case['name']
    assert R.frame_share(case['frames'], f64[0], gauss[0]).max() <= 1, case['name']
    assert abs(float(tot[c][i]) - case['score']) <= 1e-5 * max(1.0, abs(case['score'])), case['name']


@pytest.mark.parametrize('variant', ['tc6', 'ffma1', 'tree'])
def test_traced_job_replays_in_float64(native, variant):
  """A traced job under a non-model pair, replayed step by step in float64 (test_gpu_step_replay.py's check)."""
  pair, c, u = PAIRS[0], 0, 1
  if variant == 'tree':
    w, key = load_weights('model_small.npz'), 'small'
    kw = dict(beam_size=6, look_ahead=2, test_iteration=1)
    xs = utterances(64, 1150, [24, 30])
  else:
    w, key = load_weights('model_toy100.npz'), 'toy'
    kw = dict(beam_size=10, look_ahead=1, test_iteration=2, **TOY_VARIANTS[variant])
    xs = [x[:50] for x in toy_utterances()[0][6:10]]
  model = plain_model(native, key, w, own_pair(w))
  (labels, _, _, _), dbg = model.predict_sweep(xs, PAIRS, n_best=1, trace_utt=c * len(xs) + u, **kw)
  job = c * len(xs) + u
  rp = R.Replay(R.Model(with_pair(w, pair)), xs[u], kw['beam_size'], kw['look_ahead'], kw['test_iteration'],
                dbg['win'], dbg['score'], dbg['off'], 0, 0, mean0=model.constants()[0])
  final = dict(best_mean=dbg['best_mean'], best_hidden=dbg['best_hidden'], best_blocks=dbg['best_blocks'],
               final_k=dbg['final_k'][job], final_scores=dbg['final_scores'][job])
  R.check(rp, R.INC_RTOL, labels=labels[u][c][0].tolist(), final=final, state_tol=R.STATE_TOL, worst={})


def test_sweep_with_one_pair_spilling_and_another_fitting(native, monkeypatch):
  """One sweep whose jobs of the same utterances partly outgrow the shared-memory tree (status -5, decoded by the
  spill kernel's second queue) and partly fit: a huge crp_alpha opens many clusters, a tiny one few.  Which pairs
  outgrow it is read from plain calls without the spill kernel; the test needs both kinds."""
  from uisrnn_b200.synth import synth_utt
  w = load_weights('model_small.npz')
  xs = [synth_utt(1500 + i, n_frames=24, dim=64, n_spk=6, noise=0.5)[0] for i in range(2)]
  pairs = [(1e-9, 0.01), (1e-3, 0.5), (1.0, 0.5), (1e3, 0.5), (1e9, 0.99)]
  kw = dict(beam_size=8, look_ahead=3, test_iteration=1, kcap=32)
  check_sweep(native, 'small', w, xs, pairs, **kw)
  monkeypatch.setenv('UISRNN_B200_TREE_SPILL', '0')
  fits = []
  for pair in pairs:
    try:
      plain_model(native, 'small', w, pair).predict(xs, **kw)
      fits.append(True)
    except native.NativeError as err:
      assert err.code == native.UIS_ERR_CAPACITY
      fits.append(False)
  assert any(fits) and not all(fits), fits


@pytest.mark.parametrize('variant', ['ffma1', 'tree'])
def test_predict_sweep_past_4096_steps(native, variant):
  """Decodes longer than the default 4096-entry log tables (4400 frames of alternating speakers)."""
  from uisrnn_b200.synth import synth_utt
  w = load_weights('model_small.npz')
  xs = [synth_utt(7305, n_frames=4400, dim=64, n_spk=2, mean_run=1, noise=0.08)[0]]
  kw = dict(beam_size=4, look_ahead=1, test_iteration=1, engine=1, lanes=1, cluster=-1) if variant == 'ffma1' else \
      dict(beam_size=3, look_ahead=2, test_iteration=1)
  check_sweep(native, 'small', w, xs, [own_pair(w)] + PAIRS, n_best=2, **kw)


@pytest.mark.parametrize('spill', ['tree', 'spill'])
def test_tree_kernel_sweep(native, monkeypatch, spill):
  if spill == 'spill':
    monkeypatch.setenv('UISRNN_B200_TREE_SPILL', 'force')
  w = load_weights('model_small.npz')
  xs = utterances(64, 700, [40, 33, 25])
  pairs = [own_pair(w)] + PAIRS
  labels = check_sweep(native, 'small', w, xs, pairs, beam_size=8, look_ahead=2, test_iteration=2)
  # (these clean utterances decode to the same labels under every pair: the scores tell the configs apart)
  distinct(plain_model(native, 'small', w, own_pair(w)), xs, pairs, labels_too=False, beam_size=8, look_ahead=2,
           test_iteration=2)
  om = uis_oracle.OracleModel(with_pair(w, pairs[2]))
  assert labels[0][2][0].tolist() == uis_oracle.predict_single(om, xs[0], beam_size=8, look_ahead=2, test_iteration=2)


SHAPES = {'depth2': ('model_small_d2.npz', dict(engine=1, lanes=1, cluster=-1)),
          'h1024': ((1024, 512, 1), dict(engine=1)), 'padded': ((96, 40, 1), dict(engine=1, lanes=2, cluster=-1)),
          'beam64': ('model_small.npz', dict(engine=1, lanes=1, cluster=-1, beam_size=64))}


@pytest.mark.parametrize('shape', list(SHAPES))
def test_shapes_and_wide_beams(native, shape):
  key, kw = SHAPES[shape]
  w = load_weights(key) if isinstance(key, str) else random_weights(key[0], key[1], key[2], seed=5)
  D = int(np.asarray(w['w2']).shape[0])
  xs = utterances(D, 800, [36, 20, 28])
  kw = dict(dict(beam_size=10, look_ahead=1, test_iteration=2), **kw)
  check_sweep(native, shape, w, xs, [own_pair(w)] + PAIRS, n_best=4, **kw)


def test_bounds_and_nbest_compose_with_sweep(native):
  w = load_weights('model_small.npz')
  xs = utterances(64, 900, [30, 26, 0, 22])
  check_sweep(native, 'small', w, xs, PAIRS, n_best=5, beam_size=10, look_ahead=1, test_iteration=2,
              max_speakers=[3, 2, 0, 4], min_speakers=[2, 0, 0, 3], engine=1, lanes=1, cluster=-1)
  model = plain_model(native, 'small', w, own_pair(w))
  labels, scores, speakers, count = model.predict_sweep(xs, PAIRS, n_best=5, max_speakers=[3, 2, 0, 4])
  assert all(count[c][2] == 0 and np.isinf(scores[c][2]).all() for c in range(len(PAIRS)))  # the empty utterance
  assert all(labels[u][c].max() < b for c in range(len(PAIRS)) for u, b in ((0, 3), (1, 2), (3, 4)))


def test_decode_in_groups_equals_one_group(native, monkeypatch):
  w = load_weights('model_small.npz')
  xs = utterances(64, 950, [40, 30, 35, 20, 25])
  model = plain_model(native, 'small', w, own_pair(w))
  kw = dict(beam_size=10, look_ahead=1, test_iteration=2, engine=1, lanes=1, cluster=-1, n_best=2)
  whole = model.predict_sweep(xs, PAIRS, **kw)
  monkeypatch.setenv('UISRNN_B200_MAX_ROWS', '60')
  grouped = model.predict_sweep(xs, PAIRS, **kw)
  assert model.stats()['groups'] > 1
  for u in range(len(xs)):
    assert np.array_equal(whole[0][u], grouped[0][u])
  for a, b in zip(whole[1:], grouped[1:]):
    assert np.array_equal(a, b)


def test_one_pair_sweep_at_model_values_equals_plain_call(native):
  w = load_weights('model_toy100.npz')
  xs = [x[:50] for x in toy_utterances()[0][:5]]
  model = plain_model(native, 'toy', w, own_pair(w))
  for kw in (dict(), dict(engine=1, lanes=1, cluster=-1), dict(engine=2, lanes=6)):
    lab, sc, sp, cnt = model.predict(xs, n_best=2, **kw)
    labels, scores, speakers, count = model.predict_sweep(xs, [own_pair(w)], n_best=2, **kw)
    assert all(np.array_equal(labels[u][0], lab[u]) for u in range(len(xs)))
    assert np.array_equal(scores[0], sc) and np.array_equal(speakers[0], sp) and np.array_equal(count[0], cnt)


def test_device_entry_on_a_side_stream(native):
  import torch
  w = load_weights('model_small.npz')
  xs = utterances(64, 990, [30, 22, 27])
  model = plain_model(native, 'small', w, own_pair(w))
  C, k, U = len(PAIRS), 3, len(xs)
  kw = dict(beam_size=10, look_ahead=1, test_iteration=2, engine=1, lanes=2, cluster=-1)
  host = model.predict_sweep(xs, PAIRS, n_best=k, **kw)
  off = np.concatenate([[0], np.cumsum([len(x) for x in xs])]).astype(np.int64)
  x = torch.from_numpy(np.concatenate(xs).astype(np.float32)).cuda()
  lab = torch.full((C, k, int(off[-1])), -7, dtype=torch.int32, device='cuda')
  scores = torch.empty((C, U, k), dtype=torch.float32, device='cuda')
  spk = torch.empty((C, U, k), dtype=torch.int32, device='cuda')
  cnt = torch.empty((C, U), dtype=torch.int32, device='cuda')
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    model.predict_device_sweep(x.data_ptr(), off, lab.data_ptr(), scores.data_ptr(), PAIRS, n_best=k,
                               speakers_ptr=spk.data_ptr(), count_ptr=cnt.data_ptr(), stream=side.cuda_stream, **kw)
  side.synchronize()
  lab = lab.cpu().numpy()
  for u in range(U):
    assert np.array_equal(lab[:, :, off[u]:off[u + 1]], host[0][u])
  assert np.array_equal(scores.cpu().numpy(), host[1]) and np.array_equal(spk.cpu().numpy(), host[2])
  assert np.array_equal(cnt.cpu().numpy(), host[3])


@pytest.mark.parametrize('variant', ['tc6', 'ffma1', 'tree'])
def test_traced_job_equals_traced_plain_call(native, variant):
  """The step taps of job c * U + u are those of utterance u on a model created with pair c (same kernel)."""
  if variant == 'tree':
    w, key, kw = load_weights('model_small.npz'), 'small', dict(beam_size=6, look_ahead=2, test_iteration=1)
    xs = utterances(64, 1100, [24, 30])
  else:
    w, key, kw = load_weights('model_toy100.npz'), 'toy', dict(beam_size=10, look_ahead=1, test_iteration=2,
                                                              **TOY_VARIANTS[variant])
    xs = [x[:40] for x in toy_utterances()[0][:4]]
  pair, c, u = PAIRS[1], 1, 1
  sweep = plain_model(native, key, w, own_pair(w))
  _, bufs = sweep.predict_sweep(xs, PAIRS, n_best=1, trace_utt=c * len(xs) + u, **kw)
  _, want = plain_model(native, key, w, pair).predict(xs, trace_utt=u, **kw)
  for name in ('win', 'score', 'off', 'best_mean', 'best_hidden', 'best_blocks'):
    assert np.array_equal(bufs[name], want[name]), name
  assert np.array_equal(bufs['final_scores'].reshape(len(PAIRS), len(xs), -1)[c], want['final_scores'])
  assert np.array_equal(bufs['final_k'].reshape(len(PAIRS), len(xs))[c], want['final_k'])


def score_labels(rng, lengths, k):
  out = []
  for n in lengths:
    seen = {}
    out.append(np.array([seen.setdefault(int(v), len(seen)) for v in rng.integers(0, k, n)], np.int32))
  return out


@pytest.mark.parametrize('key', ['model_small.npz', 'model_toy100.npz', 'depth2'])
def test_score_sweep_equals_plain_score(native, key):
  w = load_weights('model_small_d2.npz' if key == 'depth2' else key)
  D = int(np.asarray(w['w2']).shape[0])
  xs = utterances(D, 1200, [50, 0, 37, 61])
  labs = score_labels(np.random.default_rng(3), [len(x) for x in xs], 4)
  pairs = [own_pair(w)] + PAIRS
  model = plain_model(native, key, w, own_pair(w))
  tot, inc = model.score_sweep(xs, labs, pairs, per_frame=True)
  cols = model.stats()['gru_columns']
  assert model.stats()['utterances'] == len(xs) * len(pairs)
  for c, pair in enumerate(pairs):
    ref = plain_model(native, key, w, pair)
    want, want_inc = ref.score(xs, labs, per_frame=True)
    assert np.array_equal(tot[c].view(np.uint32), want.view(np.uint32)), pair
    assert all(np.array_equal(a[c], b) for a, b in zip(inc, want_inc))
    assert ref.stats()['gru_columns'] == cols  # the chain kernel ran once for the whole sweep
  assert len({tuple(row) for row in tot.tolist()}) == len(pairs)


def test_score_sweep_long_logtot_tables_and_device_entry(native):
  """More than 4096 turns: the per-config logtot rows grow past the default table."""
  import torch
  w = load_weights('model_small.npz')
  xs = utterances(64, 1300, [4400, 300])
  labs = [np.arange(4400, dtype=np.int32) % 2, np.zeros(300, np.int32)]
  model = plain_model(native, 'small', w, own_pair(w))
  tot, inc = model.score_sweep(xs, labs, PAIRS, per_frame=True)
  for c, pair in enumerate(PAIRS):
    want, want_inc = plain_model(native, 'small', w, pair).score(xs, labs, per_frame=True)
    assert np.array_equal(tot[c], want) and all(np.array_equal(a[c], b) for a, b in zip(inc, want_inc))
  off = np.array([0, 4400, 4700], np.int64)
  x = torch.from_numpy(np.concatenate(xs).astype(np.float32)).cuda()
  lab = torch.from_numpy(np.concatenate(labs)).cuda()
  sc = torch.empty((len(PAIRS), 2), dtype=torch.float32, device='cuda')
  fr = torch.empty((len(PAIRS), 4700), dtype=torch.float32, device='cuda')
  model.score_device_sweep(x.data_ptr(), off, lab.data_ptr(), sc.data_ptr(), PAIRS, frame_ptr=fr.data_ptr())
  torch.cuda.synchronize()
  assert np.array_equal(sc.cpu().numpy(), tot)
  fr = fr.cpu().numpy()
  assert all(np.array_equal(fr[:, off[u]:off[u + 1]], inc[u]) for u in range(2))


def test_uisrnn_api_sweep_on_cuda():
  from helpers import inference_args, uisrnn_from_weights
  w = load_weights('model_small.npz')
  xs = utterances(64, 1400, [30, 25])
  model = uisrnn_from_weights(w, enable_cuda=True)
  args = inference_args(beam_size=8, test_iteration=2)
  got = model.predict(xs, args, decode_params=PAIRS)
  nb = model.predict(xs[0], args, n_best=2, decode_params=PAIRS)
  sc = model.score(xs, [[0, 1] * 15, [0] * 25], decode_params=PAIRS)
  native_before = model._native  # pylint: disable=protected-access
  for c, pair in enumerate(PAIRS):
    ref = uisrnn_from_weights(with_pair(w, pair), enable_cuda=True)
    assert got[c] == ref.predict(xs, args)
    assert nb[c].labels[0] == ref.predict(xs[0], args)
    assert sc[c] == ref.score(xs, [[0, 1] * 15, [0] * 25])
  model.predict(xs, args, decode_params=PAIRS)
  assert model._native is native_before  # pylint: disable=protected-access
  assert own_pair(w) == (model.crp_alpha, model.transition_bias)


def test_c_abi_rejects_bad_params(native):
  w = load_weights('model_small.npz')
  model = plain_model(native, 'small', w, own_pair(w))
  lib = native.load_library()
  x = np.zeros((4, 64))
  ptrs = (ctypes.c_void_p * 1)(x.ctypes.data)
  lens = np.array([4], np.int64)
  lab = np.zeros(4 * 8, np.int32)
  lptr = (ctypes.c_void_p * 1)(lab.ctypes.data)
  scores = np.zeros(8, np.float32)
  nb = native.NBestOut(ctypes.cast(lptr, ctypes.POINTER(ctypes.c_void_p)), None,
                       scores.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), None, None)
  opts = model._opts(10, 1, 1, 0, 0)  # pylint: disable=protected-access
  dbl = ctypes.POINTER(ctypes.c_double)
  cases = [(0, [1.0], [0.5], 'count'), (2, [1.0, -1.0], [0.5, 0.5], 'pair 1'), (1, [np.nan], [0.5], 'pair 0'),
           (2, [1.0, 1.0], [0.5, 1.0], 'pair 1'), (1, [1.0], [np.inf], 'pair 0')]
  for count, a, b, text in cases:
    a, b = np.array(a, np.float64), np.array(b, np.float64)
    dp = native.DecodeParams(count, a.ctypes.data_as(dbl), b.ctypes.data_as(dbl))
    rc = lib.uis_predict_sweep(model._h, ctypes.cast(ptrs, ctypes.POINTER(ctypes.c_void_p)),  # pylint: disable=protected-access
                               lens.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), 1, ctypes.byref(opts), None, None,
                               None, None, 1, ctypes.byref(nb), ctypes.byref(dp))
    assert rc == native.UIS_ERR_INVALID and text in lib.uis_last_error().decode()
    rc = lib.uis_score_sweep(model._h, ctypes.cast(ptrs, ctypes.POINTER(ctypes.c_void_p)),  # pylint: disable=protected-access
                             lens.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), 1,
                             ctypes.cast(lptr, ctypes.POINTER(ctypes.c_void_p)),
                             scores.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), None, None, ctypes.byref(dp))
    assert rc == native.UIS_ERR_INVALID and text in lib.uis_last_error().decode()
  a, b = np.ones(2, np.float64), np.full(2, 0.5)
  dp = native.DecodeParams(2, a.ctypes.data_as(dbl), b.ctypes.data_as(dbl))
  rc = lib.uis_predict_sweep(model._h, ctypes.cast(ptrs, ctypes.POINTER(ctypes.c_void_p)),  # pylint: disable=protected-access
                             lens.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), 2 ** 30 + 1, ctypes.byref(opts), None,
                             None, None, None, 1, ctypes.byref(nb), ctypes.byref(dp))
  assert rc == native.UIS_ERR_INVALID and 'INT_MAX' in lib.uis_last_error().decode()
