"""Lists larger than the device: every predict and score entry point runs a list whose workspace does not fit in
groups of whole utterances, one after the other.  UISRNN_B200_MAX_ROWS forces the group size (the only way a test may
force groups: nothing here fills the shared device's memory).  For every entry point and three limits -- about one
utterance per group, a few groups, and a limit smaller than one utterance -- the outputs must equal those of the call
run at once bit for bit, and stats()['groups'] must count the groups that the cut rule gives.

The models run kernels whose results do not depend on the other utterances of a call (the FFMA beam kernel at one lane
per CTA, the look-ahead tree kernels, the score kernels), so that a group, planned on its own, must give the same bits
as the whole call."""
import warnings

import numpy as np
import pytest
import torch

from helpers import inference_args, load_weights
from test_gpu_tensor_inputs import cuda_model, f32_bits, random_ids, synth

pytestmark = pytest.mark.gpu

# empty utterances at the start, in the middle and at the end of groups
LENGTHS = [0, 37, 12, 0, 50, 1, 0, 29, 44, 0, 18, 0]
PAIRS = [(0.5, 0.3), (2.0, 0.7)]


def cut(lengths, max_rows):
  """Groups of consecutive whole utterances of at most max_rows frames (an utterance longer: a group of its own)."""
  off = np.concatenate([[0], np.cumsum(lengths)])
  groups, u0 = 0, 0
  while u0 < len(lengths):
    u1 = u0 + 1
    while u1 < len(lengths) and off[u1 + 1] - off[u0] <= max_rows:
      u1 += 1
    groups, u0 = groups + 1, u1
  return groups


def limits(lengths):
  """(max_rows, groups): about one utterance per group, a few groups, and a limit below the shortest utterance."""
  total, longest = sum(lengths), max(lengths)
  shortest = min(n for n in lengths if n > 0)
  out = [(longest, cut(lengths, longest)), (total // 3 + 1, cut(lengths, total // 3 + 1)),
         (max(1, shortest - 1), cut(lengths, max(1, shortest - 1)))]
  assert out[0][1] > 3 and 1 < out[1][1] < out[0][1] and out[2][1] >= sum(n > 0 for n in lengths)
  return out


def grouped(monkeypatch, native, lengths, call, same):
  """call() at once, then under each limit: same(whole, got) and the stats' group count."""
  monkeypatch.delenv('UISRNN_B200_MAX_ROWS', raising=False)
  whole = call()
  st = native.stats()
  assert st['groups'] == 1, st
  for max_rows, groups in limits(lengths):
    monkeypatch.setenv('UISRNN_B200_MAX_ROWS', str(max_rows))
    got = call()
    gst = native.stats()
    assert gst['groups'] == groups, (max_rows, gst)
    for key in ('utterances', 'frames', 'gru_columns'):
      assert gst[key] == st[key], (key, max_rows, gst, st)
    same(whole, got)
  monkeypatch.delenv('UISRNN_B200_MAX_ROWS')


def bits(a):
  if isinstance(a, torch.Tensor):
    a = a.detach().cpu().numpy()
  return f32_bits(a) if np.asarray(a).dtype.kind == 'f' else np.asarray(a)


def same_tree(a, b):
  """Bit-identical nested outputs (lists, tuples, NBest / FrameScores, ndarrays, tensors, floats)."""
  if isinstance(a, (list, tuple)):
    assert type(a) is type(b) and len(a) == len(b)
    for x, y in zip(a, b):
      same_tree(x, y)
  elif isinstance(a, (float, np.floating)):
    assert f32_bits(a) == f32_bits(b)
  else:
    assert np.array_equal(bits(a), bits(b))


def as_tensors(xs):
  return [torch.from_numpy(x).float().cuda() for x in xs]


# ---------------------------------------------------------------------------------------------------------- score


@pytest.mark.parametrize('key', [('model_small.npz',), (None, 100, 37), (None, 1024, 512, 2)],
                         ids=['small', 'dim37', 'deep1024x512'])
def test_score_ndarrays(monkeypatch, key):
  model = cuda_model(*key)
  xs = synth(model.observation_dim, 40, LENGTHS)
  rng = np.random.default_rng(41)
  labels = [rng.integers(0, 4, n).tolist() for n in LENGTHS]
  native = model._native_model()  # pylint: disable=protected-access
  for kw in (dict(), dict(per_frame=True), dict(decode_params=PAIRS), dict(per_frame=True, decode_params=PAIRS)):
    grouped(monkeypatch, native, LENGTHS, lambda: model.score(xs, labels, **kw), same_tree)


@pytest.mark.parametrize('key', [('model_small.npz',), (None, 100, 37), (None, 1024, 512, 2)],
                         ids=['small', 'dim37', 'deep1024x512'])
def test_score_tensors(monkeypatch, key):
  """int64 CUDA ids (negative and beyond 32 bits: renamed on the device, group by group) and host labels."""
  model = cuda_model(*key)
  xs = synth(model.observation_dim, 42, LENGTHS)
  ts = as_tensors(xs)
  rng = np.random.default_rng(43)
  ids = [torch.from_numpy(random_ids(rng, n, 1 + u % 5)).cuda() for u, n in enumerate(LENGTHS)]
  host = [['spk%d' % v for v in i.cpu().tolist()] for i in ids]
  native = model._native_model()  # pylint: disable=protected-access
  for labels in (ids, host):
    for kw in (dict(), dict(per_frame=True), dict(per_frame=True, decode_params=PAIRS)):
      grouped(monkeypatch, native, LENGTHS, lambda: model.score(ts, labels, **kw), same_tree)
  # the tensor call equals the ndarray call, grouped or not
  monkeypatch.setenv('UISRNN_B200_MAX_ROWS', '1')
  same_tree(model.score(ts, ids, decode_params=PAIRS)[1].cpu().numpy(),
            np.asarray(model.score([t.double().cpu().numpy() for t in ts], host, decode_params=PAIRS)[1], np.float32))


@pytest.fixture(scope='module')
def small_native():
  from uisrnn_b200 import native
  return native.NativeModel(load_weights('model_small.npz'))


def device_rows(xs, D):
  off = np.zeros(len(xs) + 1, np.int64)
  np.cumsum([len(x) for x in xs], out=off[1:])
  return torch.from_numpy(np.concatenate(xs).astype(np.float32).reshape(-1, D)).cuda(), off


def test_score_device_and_sweep(monkeypatch, small_native):
  from uisrnn_b200.uisrnn import canonical_labels
  m = small_native
  xs = synth(m.D, 44, LENGTHS)
  x, off = device_rows(xs, m.D)
  rng = np.random.default_rng(45)
  canon = np.concatenate([canonical_labels(rng.integers(0, 5, n)) for n in LENGTHS]).astype(np.int32)
  lab = torch.from_numpy(canon).cuda()
  rows, U = int(off[-1]), len(LENGTHS)

  def plain():
    scores, frames = torch.full((U,), -1.0, device='cuda'), torch.full((rows,), -1.0, device='cuda')
    m.score_device(x.data_ptr(), off, lab.data_ptr(), scores.data_ptr(), frames.data_ptr())
    return scores.cpu().numpy(), frames.cpu().numpy()

  def sweep():
    scores, frames = torch.full((2, U), -1.0, device='cuda'), torch.full((2, rows), -1.0, device='cuda')
    m.score_device_sweep(x.data_ptr(), off, lab.data_ptr(), scores.data_ptr(), PAIRS, frame_ptr=frames.data_ptr())
    return scores.cpu().numpy(), frames.cpu().numpy()

  grouped(monkeypatch, m, LENGTHS, plain, same_tree)
  grouped(monkeypatch, m, LENGTHS, sweep, same_tree)


def test_score_call_returns_before_its_groups_run(monkeypatch):
  """A grouped tensor score() enqueues every group on torch's current stream and returns: behind a long sleep on that
  stream, an event recorded right after the call has not completed."""
  model = cuda_model('model_small.npz')
  xs = synth(model.observation_dim, 46, LENGTHS)
  ts = as_tensors(xs)
  rng = np.random.default_rng(47)
  ids = [torch.from_numpy(random_ids(rng, n, 4)).cuda() for n in LENGTHS]
  want = model.score(ts, ids, decode_params=PAIRS)
  monkeypatch.setenv('UISRNN_B200_MAX_ROWS', str(max(LENGTHS)))
  model.score(ts, ids, decode_params=PAIRS)  # warm-up: the workspace of the largest group, the tables
  torch.cuda.synchronize()
  stream = torch.cuda.Stream()
  with torch.cuda.stream(stream):
    torch.cuda._sleep(500_000_000)  # pylint: disable=protected-access
    got = model.score(ts, ids, decode_params=PAIRS)
    done = torch.cuda.Event()
    done.record()
  assert not done.query()
  assert model._native_model().stats()['groups'] == cut(LENGTHS, max(LENGTHS))  # pylint: disable=protected-access
  same_tree([g.cpu().numpy() for g in got], [w.cpu().numpy() for w in want])


# -------------------------------------------------------------------------------------------------------- predict


@pytest.mark.parametrize('key', [('model_small.npz',), (None, 100, 37), (None, 1024, 512, 2)],
                         ids=['small', 'dim37', 'deep1024x512'])
def test_predict_tensors(monkeypatch, key):
  """Tensor predict() with n_best, per-utterance bounds and decode_params."""
  model = cuda_model(*key)
  lengths = LENGTHS if key[0] else [n // 2 for n in LENGTHS]  # (the deep model: shorter utterances)
  xs = synth(model.observation_dim, 48, lengths)
  ts = as_tensors(xs)
  native = model._native_model()  # pylint: disable=protected-access
  args = inference_args(beam_size=4, test_iteration=2)
  mx = [(2, 0, 3, 1)[u % 4] for u in range(len(lengths))]
  mn = [(1, 0, 2, 0)[u % 4] for u in range(len(lengths))]
  for kw in (dict(), dict(n_best=3), dict(n_best=2, max_speakers=mx, min_speakers=mn),
             dict(n_best=2, decode_params=PAIRS, max_speakers=mx)):
    with warnings.catch_warnings():  # (the min_speakers warning of the bounded calls)
      warnings.simplefilter('ignore')
      grouped(monkeypatch, native, lengths, lambda: model.predict(ts, args, **kw), same_tree)


@pytest.mark.parametrize('look_ahead,spill', [(2, None), (3, None), (2, 'force')])
def test_predict_look_ahead(monkeypatch, look_ahead, spill):
  model = cuda_model('model_small.npz')
  xs = synth(model.observation_dim, 50 + look_ahead, LENGTHS)
  ts = as_tensors(xs)
  native = model._native_model()  # pylint: disable=protected-access
  if spill:
    monkeypatch.setenv('UISRNN_B200_TREE_SPILL', spill)  # every tree from the device-memory arena
  args = inference_args(beam_size=3, look_ahead=look_ahead, test_iteration=1)
  grouped(monkeypatch, native, LENGTHS, lambda: model.predict(ts, args, n_best=2), same_tree)


def test_predict_device_sweep_on_a_side_stream(monkeypatch, small_native):
  m = small_native
  xs = synth(m.D, 52, LENGTHS)
  x, off = device_rows(xs, m.D)
  rows, U, k, C = int(off[-1]), len(LENGTHS), 3, len(PAIRS)
  side = torch.cuda.Stream()

  def call():
    lab = torch.full((C, k, rows), -9, dtype=torch.int32, device='cuda')
    sc = torch.full((C, U, k), -9.0, device='cuda')
    sp = torch.full((C, U, k), -9, dtype=torch.int32, device='cuda')
    cnt = torch.full((C, U), -9, dtype=torch.int32, device='cuda')
    torch.cuda.synchronize()
    m.predict_device_sweep(x.data_ptr(), off, lab.data_ptr(), sc.data_ptr(), PAIRS, beam_size=5, test_iteration=2,
                           stream=side.cuda_stream, n_best=k, speakers_ptr=sp.data_ptr(), count_ptr=cnt.data_ptr(),
                           max_speakers=[3] * U, engine=1, lanes=1, cluster=-1)
    side.synchronize()
    return [t.cpu().numpy() for t in (lab, sc, sp, cnt)]

  grouped(monkeypatch, m, LENGTHS, call, same_tree)
  # every output was written: the empty utterances return no hypothesis
  lab, sc, sp, cnt = call()
  for u, n in enumerate(LENGTHS):
    assert (cnt[:, u] == 0).all() == (n == 0) and (cnt[:, u] >= 0).all()
    if n == 0:
      assert np.isinf(sc[:, u]).all() and (sp[:, u] == 0).all()
  assert (lab[:, 0] >= 0).all()

