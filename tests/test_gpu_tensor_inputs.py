"""predict() and score() of torch CUDA tensors: bit for bit what the ndarray calls give for the same values, on every
kernel the planner picks, with bounds, N-best and decode_params; the device renaming and chain plan of
uis_score_device_ids against canonical_labels and the host plan; no synchronisation and stream ordering."""
import numpy as np
import pytest
import torch

from helpers import inference_args, load_weights, uisrnn_from_weights
from test_gpu_large_models import large_model, utterances

pytestmark = pytest.mark.gpu

_MODELS = {}


def cuda_model(name, H=None, D=None, depth=1):
  """A CUDA UISRNN of a golden fixture (name) or of large_model(H, D, depth)."""
  key = (name, H, D, depth)
  if key not in _MODELS:
    w = load_weights(name) if name else large_model(H, D, depth, seed=9000 + H + D + depth)
    _MODELS[key] = uisrnn_from_weights(w, enable_cuda=True)
  return _MODELS[key]


def synth(D, seed, lengths):
  return [np.asarray(x, np.float64) for x in utterances(D, seed, lengths)]


def as_tensors(xs, dtype, strided):
  """The rows as CUDA tensors of `dtype` (strided: transposed views), and the float64 ndarrays of their exact values."""
  out = []
  for x in xs:
    t = torch.from_numpy(np.ascontiguousarray(x.T) if strided else x).cuda().to(dtype)
    out.append(t.t() if strided else t)
  return out, [t.double().cpu().numpy() for t in out]


def same_labels(got, want):
  assert isinstance(got, torch.Tensor) and got.dtype == torch.int64 and got.is_cuda
  assert got.cpu().tolist() == list(want)


def same_nbest(got, want):
  assert got.labels.cpu().tolist() == [list(l) for l in want.labels]
  assert got.scores.dtype == torch.float32 and got.speakers.dtype == torch.int32
  assert np.array_equal(got.scores.cpu().numpy().view(np.uint32), np.asarray(want.scores, np.float32).view(np.uint32))
  assert got.speakers.cpu().tolist() == list(want.speakers)


def compare_predict(model, xs, args, dtype=torch.float32, strided=False, expect=None, **kw):
  """predict() of the tensors against predict() of their float64 values; `expect` checks the kernel the call ran."""
  ts, arrays = as_tensors(xs, dtype, strided)
  got = model.predict(ts, args, **kw)
  if expect:
    expect(model._native_model().stats())  # pylint: disable=protected-access
  want = model.predict(arrays, args, **kw)
  swept = kw.get('decode_params') is not None
  for g_row, w_row in zip(got, want) if swept else [(got, want)]:
    assert len(g_row) == len(w_row)
    for g, w in zip(g_row, w_row):
      if kw.get('n_best'):
        same_nbest(g, w)
      else:
        same_labels(g, w)


KERNELS = {
    # name: (model key, lengths, expected stats)
    'tensor_cores': (('model_toy100.npz',), [6 + i % 9 for i in range(140)], lambda s: s['engine'] == 2),
    'ffma': (('model_toy100.npz',), [8 + i % 7 for i in range(100)], lambda s: s['engine'] == 1 and s['cluster'] == 1),
    'cluster': (('model_toy100.npz',), [20 + i for i in range(12)], lambda s: s['cluster'] in (2, 4, 8)),
    'stationary': (('model_toy100.npz',), [30, 1, 25], lambda s: s['cluster'] == 32),
    'small_ffma': (('model_small.npz',), [40, 0, 1, 33, 17], lambda s: s['engine'] == 1),
    'depth2': (('model_small_d2.npz',), [30, 12, 1, 0, 25], None),
    'padded': ((None, 100, 40), [35, 0, 22, 1], None),
}


@pytest.mark.parametrize('kernel', sorted(KERNELS))
@pytest.mark.parametrize('dtype,strided', [(torch.float32, False), (torch.float64, True), (torch.float16, False),
                                           (torch.bfloat16, True)])
def test_predict_bit_for_bit(kernel, dtype, strided):
  key, lengths, expect = KERNELS[kernel]
  model = cuda_model(*key)
  xs = synth(model.observation_dim, 100 + len(lengths), lengths)
  check = (lambda s: None if expect(s) else pytest.fail('{} did not run: {}'.format(kernel, s))) if expect else None
  compare_predict(model, xs, inference_args(beam_size=4, test_iteration=2), dtype, strided, expect=check)


@pytest.mark.parametrize('kernel', ['tensor_cores', 'stationary', 'small_ffma', 'padded'])
def test_predict_bounds_nbest_and_sweeps(kernel):
  key, lengths, _ = KERNELS[kernel]
  model = cuda_model(*key)
  xs = synth(model.observation_dim, 300 + len(lengths), lengths)
  args = inference_args(beam_size=5, test_iteration=1)
  compare_predict(model, xs, args, n_best=3)
  compare_predict(model, xs, args, max_speakers=2, min_speakers=1)
  compare_predict(model, xs, args, decode_params=[(0.5, 0.3), (2.0, 0.7)], n_best=2)
  compare_predict(model, xs, args, decode_params=[(1.5, 0.4)], max_speakers=[3] * len(xs), min_speakers=2)


def test_predict_look_ahead_2_and_single_tensors():
  model = cuda_model('model_small.npz')
  xs = synth(model.observation_dim, 400, [18, 1, 0, 11])
  compare_predict(model, xs, inference_args(beam_size=3, look_ahead=2, test_iteration=2))
  compare_predict(model, xs, inference_args(beam_size=3, look_ahead=2, test_iteration=1), torch.float16, n_best=2)
  args = inference_args(beam_size=4, test_iteration=2)
  for x in xs:
    t = torch.from_numpy(x).cuda()
    same_labels(model.predict(t, args), model.predict(x, args))
    same_labels(model.predict_single(t, args), model.predict_single(x, args))
    same_nbest(model.predict(t, args, n_best=2), model.predict(x, args, n_best=2))
  x32 = torch.from_numpy(xs[0]).float().cuda().requires_grad_()
  same_labels(model.predict(x32, args), model.predict(x32.detach().double().cpu().numpy(), args))


def test_predict_input_errors():
  model = cuda_model('model_small.npz')
  args = inference_args(beam_size=2, test_iteration=1)
  D = model.observation_dim
  with pytest.raises(TypeError):
    model.predict([torch.zeros(3, D, device='cuda'), np.zeros((3, D))], args)
  with pytest.raises(TypeError):
    model.predict([torch.zeros(3, D, device='cuda'), torch.zeros(3, D, device='cuda', dtype=torch.float64)], args)
  with pytest.raises(TypeError):
    model.predict(torch.zeros(3, D, device='cuda', dtype=torch.int32), args)
  with pytest.raises(ValueError, match='2-dim'):
    model.predict(torch.zeros(3, device='cuda'), args)
  with pytest.raises(ValueError, match='observation_dim'):
    model.predict(torch.zeros(3, D + 1, device='cuda'), args)
  with pytest.raises(ValueError, match="model's device"):
    model.predict(torch.zeros(3, D), args)
  assert model.predict([], args) == []


# ---------------------------------------------------------------------------------------------------------- score


def random_ids(rng, n, k):
  """n int64 ids drawn from k random values: negatives, values >= 2^32, first appearances in no particular order."""
  pool = rng.integers(-2 ** 62, 2 ** 62, k)
  pool[0], pool[-1] = -5, 2 ** 40 + 3
  return pool[rng.integers(0, k, n)]


def f32_bits(a):
  return np.asarray(a, np.float32).view(np.uint32)


def compare_score(model, xs, ids, dtype=torch.float32, **kw):
  from uisrnn_b200.uisrnn import canonical_labels
  ts, arrays = as_tensors(xs, dtype, strided=False)
  id_tensors = [torch.from_numpy(np.asarray(i, np.int64)).cuda() for i in ids]
  got = model.score(ts, id_tensors, **kw)
  want = model.score(arrays, [canonical_labels(i) for i in ids], **kw)
  swept = kw.get('decode_params') is not None
  for g, w in zip(got, want) if swept else [(got, want)]:
    if kw.get('per_frame'):
      assert len(g) == len(w)
      for gf, wf in zip(g, w):
        assert gf.total.dim() == 0 and f32_bits(gf.total.cpu()) == f32_bits(wf.total)
        assert np.array_equal(f32_bits(gf.increments.cpu()), f32_bits(wf.increments))
    else:
      assert g.dtype == torch.float32 and g.shape == (len(xs),)
      assert np.array_equal(f32_bits(g.cpu()), f32_bits(w))
  return got


SCORE_MODELS = [('model_toy100.npz',), ('model_small.npz',), ('model_small_d2.npz',), (None, 100, 40)]


@pytest.mark.parametrize('key', SCORE_MODELS, ids=['toy', 'small', 'depth2', 'padded'])
def test_score_bit_for_bit(key):
  model = cuda_model(*key)
  rng = np.random.default_rng(7)
  lengths = [60, 0, 1, 45, 2, 33]
  xs = synth(model.observation_dim, 500, lengths)
  ids = [random_ids(rng, n, 1 + u % 5) for u, n in enumerate(lengths)]
  compare_score(model, xs, ids)
  compare_score(model, xs, ids, per_frame=True)
  compare_score(model, xs, ids, dtype=torch.bfloat16, decode_params=[(0.5, 0.2), (3.0, 0.8)])
  compare_score(model, xs, ids, dtype=torch.float64, per_frame=True, decode_params=[(0.7, 0.6)])
  # a single tensor: a 0-d score; host label sequences of any hashable values are renamed, then uploaded
  from uisrnn_b200.uisrnn import canonical_labels
  t = torch.from_numpy(xs[0]).cuda()
  names = ['spk%d' % v for v in canonical_labels(ids[0])]
  s = model.score(t, names)
  assert s.dim() == 0 and f32_bits(s.cpu()) == f32_bits(model.score(xs[0], names))
  relabelled = torch.from_numpy(canonical_labels(ids[0]) * 3 - 7).cuda()  # int32, distinct where ids[0] is
  s = model.score(t, relabelled, decode_params=[(2.0, 0.5)])
  assert len(s) == 1 and f32_bits(s[0].cpu()) == f32_bits(model.score(xs[0], ids[0], decode_params=[(2.0, 0.5)])[0])
  with pytest.raises(ValueError, match='labels for'):
    model.score([t], [torch.zeros(3, dtype=torch.int64, device='cuda')])
  with pytest.raises(TypeError, match='integer dtype'):
    model.score([t], [torch.zeros(len(xs[0]), device='cuda')])


def native_plan(m, xs, ids):
  """(scores, canonical labels, stats) of uis_score_device_ids, and the same of uis_score_device_sweep fed the
  canonical labels (the host plan)."""
  from uisrnn_b200.uisrnn import canonical_labels
  off = np.zeros(len(xs) + 1, np.int64)
  np.cumsum([len(x) for x in xs], out=off[1:])
  rows = int(off[-1])
  x = torch.from_numpy(np.concatenate(xs).astype(np.float32) if rows else np.zeros((0, m.D), np.float32)).cuda()
  idt = torch.from_numpy(np.concatenate(ids).astype(np.int64) if rows else np.zeros(0, np.int64)).cuda()
  got, lab = torch.empty(max(len(xs), 1), device='cuda'), torch.full((max(rows, 1),), -7, dtype=torch.int32, device='cuda')
  m.score_device_ids(x.data_ptr(), off, idt.data_ptr() if rows else 0, got.data_ptr(), None, labels_ptr=lab.data_ptr())
  st_dev = m.stats()
  canon = np.concatenate([canonical_labels(i) for i in ids]) if rows else np.zeros(0, np.int32)
  ct = torch.from_numpy(canon).cuda()
  want = torch.empty(max(len(xs), 1), device='cuda')
  m.score_device_sweep(x.data_ptr(), off, ct.data_ptr() if rows else 0, want.data_ptr(), None)
  st_host = m.stats()
  torch.cuda.synchronize()
  assert lab[:rows].cpu().numpy().tolist() == canon.tolist()
  assert np.array_equal(f32_bits(got[:len(xs)].cpu()), f32_bits(want[:len(xs)].cpu()))
  # (weight_passes may differ: the device plan's chain kernel runs on a grid sized from the rows, not the queue)
  for key in ('gru_columns', 'max_k', 'utterances', 'frames'):
    assert st_dev[key] == st_host[key], (key, st_dev, st_host)
  return got[:len(xs)].cpu().numpy(), st_dev


@pytest.fixture(scope='module')
def small_native():
  from uisrnn_b200 import native
  return native.NativeModel(load_weights('model_small.npz'))


def test_renaming_and_plan_edge_cases(small_native):
  m = small_native
  rng = np.random.default_rng(11)
  D = m.D
  # every frame opens a cluster: no chain is queued
  xs = synth(D, 600, [40, 7])
  distinct = rng.integers(-2 ** 62, 2 ** 62, 40)
  assert len(set(distinct.tolist())) == 40
  _, st = native_plan(m, xs, [distinct, np.arange(7) * -3])
  assert st['gru_columns'] == 0 and st['max_k'] == 40
  # one 10^5-frame single-cluster utterance
  x = synth(D, 601, [100000])
  _, st = native_plan(m, x, [np.full(100000, -(2 ** 50), np.int64)])
  assert st['gru_columns'] == 99999 and st['max_k'] == 1
  # 10^4 short utterances, random ids
  lengths = rng.integers(0, 6, 10000)
  xs = [np.asarray(rng.normal(size=(n, D)) * 0.3, np.float64) for n in lengths]
  ids = [random_ids(rng, int(n), 3) for n in lengths]
  native_plan(m, xs, ids)
  # mixed lengths and many clusters
  lengths = [300, 1, 0, 250, 2]
  native_plan(m, synth(D, 602, lengths), [random_ids(rng, n, 40) for n in lengths])
  # U = 0 and all-empty lists
  scores, st = native_plan(m, [], [])
  assert st['utterances'] == 0 and st['frames'] == 0
  scores, st = native_plan(m, [np.zeros((0, D))] * 3, [np.zeros(0, np.int64)] * 3)
  assert scores.tolist() == [0.0, 0.0, 0.0] and st['frames'] == 0


def test_score_call_does_not_synchronise(small_native):
  m = small_native
  rng = np.random.default_rng(12)
  xs = synth(m.D, 700, [300, 200, 150])
  off = np.array([0, 300, 500, 650], np.int64)
  ids = np.concatenate([random_ids(rng, n, 6) for n in (300, 200, 150)])
  x = torch.from_numpy(np.concatenate(xs).astype(np.float32)).cuda()
  idt = torch.from_numpy(ids).cuda()
  out = torch.empty(3, device='cuda')
  m.score_device_ids(x.data_ptr(), off, idt.data_ptr(), out.data_ptr(), None)  # warm-up: workspace and tables
  torch.cuda.synchronize()
  want = out.clone()
  out.fill_(-1)
  stream = torch.cuda.Stream()
  torch.cuda.synchronize()
  with torch.cuda.stream(stream):
    torch.cuda._sleep(500_000_000)  # pylint: disable=protected-access
    m.score_device_ids(x.data_ptr(), off, idt.data_ptr(), out.data_ptr(), None, stream=stream.cuda_stream)
  assert not stream.query()
  stream.synchronize()
  assert np.array_equal(f32_bits(out.cpu()), f32_bits(want.cpu()))


def test_calls_from_two_streams_are_ordered(small_native):
  m = small_native
  rng = np.random.default_rng(13)
  calls = []
  for seed, lengths in ((800, [400, 350]), (801, [90, 120, 60, 30])):
    xs = synth(m.D, seed, lengths)
    off = np.zeros(len(xs) + 1, np.int64)
    np.cumsum(lengths, out=off[1:])
    ids = np.concatenate([random_ids(rng, n, 5) for n in lengths])
    x, idt = torch.from_numpy(np.concatenate(xs).astype(np.float32)).cuda(), torch.from_numpy(ids).cuda()
    out = torch.empty(len(xs), device='cuda')
    m.score_device_ids(x.data_ptr(), off, idt.data_ptr(), out.data_ptr(), None)
    torch.cuda.synchronize()
    calls.append((x, off, idt, out.clone(), torch.full_like(out, -1)))
  s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
  torch.cuda.synchronize()
  (x1, o1, i1, w1, g1), (x2, o2, i2, w2, g2) = calls
  with torch.cuda.stream(s1):
    torch.cuda._sleep(300_000_000)  # pylint: disable=protected-access
    m.score_device_ids(x1.data_ptr(), o1, i1.data_ptr(), g1.data_ptr(), None, stream=s1.cuda_stream)
  m.score_device_ids(x2.data_ptr(), o2, i2.data_ptr(), g2.data_ptr(), None, stream=s2.cuda_stream)
  # the second call's stream waits for the first call, which waits behind the sleep: unordered, s2 would run at once
  assert not s2.query()
  torch.cuda.synchronize()
  assert np.array_equal(f32_bits(g1.cpu()), f32_bits(w1.cpu()))
  assert np.array_equal(f32_bits(g2.cpu()), f32_bits(w2.cpu()))


def test_strided_label_tensors_and_misaligned_rows():
  """A single utterance's label tensor of any strides (a column, a step slice, an expanded scalar) scores as its
  contiguous copy, and fp32 rows that start off a 16-byte boundary are copied, not read with misaligned loads."""
  model = cuda_model('model_small.npz')
  D = model.observation_dim
  rng = np.random.default_rng(21)
  x = synth(D, 900, [64])[0]
  t = torch.from_numpy(x).float().cuda()
  pairs = torch.from_numpy(np.stack([rng.integers(-9, 9, 64), random_ids(rng, 64, 5)], 1)).cuda()
  twice = torch.from_numpy(random_ids(rng, 128, 4)).cuda()
  for ids in (pairs[:, 1], twice[::2], torch.tensor([2 ** 40], device='cuda').expand(64), pairs[:, 0].int()):
    assert ids.shape == (64,)
    want = model.score(t, ids.contiguous(), per_frame=True)
    for got in (model.score(t, ids, per_frame=True), model.score([t], [ids], per_frame=True)[0]):
      assert f32_bits(got.total.cpu()) == f32_bits(want.total.cpu())
      assert np.array_equal(f32_bits(got.increments.cpu()), f32_bits(want.increments.cpu()))
  flat = torch.zeros(1 + 64 * D, device='cuda')
  shifted = flat[1:].view(64, D)
  shifted.copy_(t)
  assert shifted.is_contiguous() and shifted.data_ptr() % 16 == 4
  ids = pairs[:, 1].contiguous()
  assert f32_bits(model.score(shifted, ids).cpu()) == f32_bits(model.score(t, ids).cpu())
  args = inference_args(beam_size=4, test_iteration=2)
  same_labels(model.predict(shifted, args), model.predict(x.astype(np.float32).astype(np.float64), args))
