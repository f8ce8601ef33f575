"""score() on the GPU: the reference's neg_likelihood of given labellings (tests/golden/score_cases.npz), the float64
rescorer on every kernel shape, padded shape and depth, bit-for-bit agreement with the N-best scores of the FFMA beam
kernels, edge cases of the chain plan, call composition and validation."""
import numpy as np
import pytest

from beam_replay import path_score
from helpers import inference_args, load_weights, uisrnn_from_weights
from test_gpu_large_models import large_model, utterances
from test_score_cpu import CASES, check_case

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def native():
  from uisrnn_b200 import native as nat
  nat.load_library()
  return nat


_MODELS = {}


def cuda_model(name):
  if name not in _MODELS:
    _MODELS[name] = uisrnn_from_weights(load_weights(name), enable_cuda=True)
  return _MODELS[name]


def random_labels(rng, n, k):
  seen = {}
  return np.array([seen.setdefault(int(v), len(seen)) for v in rng.integers(0, k, n)], np.int32)


def check_rescored(w, xs, labels, got):
  ps = path_score(w, xs, [l[None] for l in labels], device='cuda')
  share = ps.share(np.asarray(got, np.float64))
  assert np.all(share <= 1), (share.max(), int(np.argmax(share)))


def test_golden_cases():
  by_model = {}
  for c in CASES:
    by_model.setdefault(c['model'], []).append(c)
  for name, cases in by_model.items():
    got = cuda_model(name).score([c['x'] for c in cases], [c['labels'] for c in cases])
    for g, c in zip(got, cases):
      check_case(g, c)


SHAPES = [(128, 64, 1), (256, 128, 1), (512, 256, 1), (1024, 512, 1), (600, 300, 1), (256, 128, 2), (256, 128, 3),
          (256, 128, 4), (512, 256, 2), (1024, 512, 2), (600, 300, 2)]


@pytest.mark.parametrize('H,D,depth', SHAPES)
def test_shapes_and_depths(native, H, D, depth):
  w = large_model(H, D, depth, seed=7000 + H + D + depth)
  m = native.NativeModel(w)
  rng = np.random.default_rng(H + depth)
  xs = utterances(D, 7100 + depth, (37, 1, 60, 0, 23))
  labels = [random_labels(rng, len(x), k) for x, k in zip(xs, (5, 1, 9, 1, 23))]
  got, frames = m.score(xs, labels, per_frame=True)
  check_rescored(w, xs, labels, got)
  st = m.stats()
  assert st['engine'] == 1 and st['gru_columns'] == sum(len(l) for l in labels) - sum(len(set(l)) for l in labels)
  for g, f in zip(got, frames):
    s = np.float32(0)
    for v in f:
      s = np.float32(s + v)
    assert s == g


@pytest.mark.parametrize('depth', [1, 2])
def test_nbest_scores_bit_for_bit(native, depth):
  name = 'model_toy100.npz' if depth == 1 else 'model_small_d2.npz'
  m = native.NativeModel(load_weights(name))
  D = m.D
  from uisrnn_b200.synth import synth_utt
  xs = [synth_utt(7200 + u, n_frames=40 + 13 * u, dim=D, n_spk=4, noise=0.06 if D == 256 else 0.08)[0]
        for u in range(6)]
  labels, scores, _, count = m.predict(xs, beam_size=10, look_ahead=1, test_iteration=1, n_best=5, engine=1,
                                       cluster=-1)
  seqs, labs, want = [], [], []
  for u, x in enumerate(xs):
    for j in range(count[u]):
      seqs.append(x)
      labs.append(labels[u][j])
      want.append(scores[u][j])
  got = m.score(seqs, labs)
  assert np.array_equal(got.view(np.uint32), np.array(want, np.float32).view(np.uint32))
  for kw in (dict(engine=2), dict(cluster=2, engine=1)) if depth == 1 else ():
    labels, scores, _, count = m.predict(xs, beam_size=10, look_ahead=1, test_iteration=1, n_best=5, **kw)
    seqs = [x for u, x in enumerate(xs) for _ in range(count[u])]
    labs = [labels[u][j] for u in range(len(xs)) for j in range(count[u])]
    got = m.score(seqs, labs)
    check_rescored(load_weights(name), seqs, labs, got)


def test_edge_cases_and_composition(native):
  import torch
  w = load_weights('model_small.npz')
  m = native.NativeModel(w)
  rng = np.random.default_rng(11)
  long = utterances(64, 7300, (4200,))[0]
  many, single = utterances(64, 7301, (300, 50))
  ragged = utterances(64, 7400, tuple(int(v) for v in rng.integers(0, 60, 1100)))
  xs = [long, many, single, long[:0]] + ragged
  from uisrnn_b200.uisrnn import canonical_labels
  labels = [np.zeros(4200, np.int32), canonical_labels(rng.permutation(np.arange(300) % 100)),
            np.arange(50, dtype=np.int32),
            np.zeros(0, np.int32)] + [random_labels(rng, len(x), 6) for x in ragged]
  assert labels[1].max() + 1 == 100
  got, frames = m.score(xs, labels, per_frame=True)
  assert got[3] == 0.0
  check_rescored(w, xs, labels, got)
  bits = got.view(np.uint32)
  # single calls, reversed order, host vs device entry point
  for i in (0, 1, 2, 3, 10, 500):
    assert m.score([xs[i]], [labels[i]]).view(np.uint32)[0] == bits[i]
  rev = m.score(xs[::-1], labels[::-1])
  assert np.array_equal(rev[::-1].view(np.uint32), bits)
  off = np.concatenate([[0], np.cumsum([len(x) for x in xs])]).astype(np.int64)
  x_dev = torch.from_numpy(np.concatenate(xs).astype(np.float32)).cuda()
  l_dev = torch.from_numpy(np.concatenate(labels).astype(np.int32)).cuda()
  s_dev = torch.empty(len(xs), dtype=torch.float32, device='cuda')
  f_dev = torch.empty(int(off[-1]), dtype=torch.float32, device='cuda')
  m.score_device(x_dev.data_ptr(), off, l_dev.data_ptr(), s_dev.data_ptr(), f_dev.data_ptr())
  torch.cuda.synchronize()
  assert np.array_equal(s_dev.cpu().numpy().view(np.uint32), bits)
  assert np.array_equal(f_dev.cpu().numpy().view(np.uint32), np.concatenate(frames).view(np.uint32))
  st = m.stats()
  assert st['max_k'] == 100 and st['utterances'] == len(xs) and st['frames'] == off[-1]


def test_uisrnn_score_and_validation(native):
  case = next(c for c in CASES if c['name'] == 's_singletons')
  model = cuda_model(case['model'])
  x, lab = case['x'], case['labels']
  cpu = uisrnn_from_weights(load_weights(case['model']))
  assert abs(model.score(x, lab) - cpu.score(x, lab)) <= 1e-5 * abs(cpu.score(x, lab))
  fs = model.score(x, ['s%d' % v for v in lab], per_frame=True)
  assert fs.total == model.score(x, lab) and fs.increments.dtype == np.float32
  m = model._native_model()  # pylint: disable=protected-access
  bad = lab.astype(np.int32).copy()
  bad[3] = bad.max() + 2
  with pytest.raises(native.NativeError) as err:
    m.score([x], [bad])
  assert err.value.code == native.UIS_ERR_INVALID and b'frame 3' in str(err.value).encode()
  with pytest.raises(ValueError):
    m.score([x], [lab[:-1]])
  with pytest.raises(ValueError):
    model.score([x, x], [lab, lab[:-1]])
  args = inference_args(beam_size=10, test_iteration=1)
  assert model.predict(x, args) is not None  # predict() still works after score calls on the same handle
