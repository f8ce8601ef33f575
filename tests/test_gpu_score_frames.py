"""score() per frame on the GPU.  Every call's per-frame increments are checked against the float64 rescore
(beam_replay.path_score(per_frame=True)) within the per-frame allowance -- one fp32 ulp of the increment plus INC_RTOL
times the frame's Gaussian term -- and every total must be the bits of the fp32 running sum of its own per-frame
increments.  A Gaussian term written to another frame's row, or a per-frame output shifted by one, leaves the totals
unchanged up to fp32 reassociation; only a per-frame check sees it.

Covered: the reference's golden cases (tests/golden/score_cases.npz, whose per-frame losses are compared too) through
the host and the device entry points; every kernel shape, depth and zero-padded shape through both; the reduce
kernel's log tables past their default 4096 entries, grown from a score call on a fresh handle and after a predict()
on the same handle; 3000 clusters in one utterance; the chain plan's edges (no chain queued, one, chains of two frames
only, more chains than the resident columns); the first-column rule; the device entry point without per-frame output,
on a side stream and with non-canonical labels; the host path's staging variants; and the N-best scores of the FFMA
beam kernel, bit for bit, at the shapes, depths, beams and lane counts test_gpu_score.py leaves out.

The worst per-frame share of each group is printed at the end of the module (pytest -s)."""
import numpy as np
import pytest

from beam_replay import frame_allowance, frame_share, path_score
from helpers import load_weights
from test_gpu_large_models import _cached, large_model, utterances
from test_gpu_score import SHAPES, random_labels
from test_score_cpu import CASES, fp32_sum

pytestmark = pytest.mark.gpu

# zero-padded shapes (run in the next larger kernel shape), as in test_gpu_parity.py
PADDED = [(100, 40, 1), (8, 2, 2), (300, 200, 1), (129, 65, 1), (512, 100, 1), (24, 16, 3)]

WORST = {}  # group -> worst per-frame share (and other measurements), printed at the end


def note(key, value):
  WORST[key] = max(WORST.get(key, value), value) if isinstance(value, float) else value


@pytest.fixture(scope='module', autouse=True)
def report():
  yield
  for k in sorted(WORST):
    print('score per frame: %-28s %s' % (k, WORST[k]))


@pytest.fixture(scope='module')
def native():
  from uisrnn_b200 import native as nat
  nat.load_library()
  return nat


def padded_model(H, D, depth):
  """test_gpu_parity.py's model of a shape that runs zero-padded."""
  rng = np.random.default_rng(1000 * H + D)
  u = lambda *s: (rng.uniform(-1, 1, size=s) / np.sqrt(H)).astype(np.float32)
  w = {'depth': depth, 'w1': u(H, H), 'b1': u(H), 'w2': u(D, H), 'b2': u(D), 'h0': u(depth, 1, H),
       'sigma2': (0.05 + 0.1 * rng.random(D)).astype(np.float32), 'transition_bias': 0.15, 'crp_alpha': 1.0}
  for l in range(depth):
    w['weight_ih_l%d' % l] = u(3 * H, D if l == 0 else H); w['weight_hh_l%d' % l] = u(3 * H, H)
    w['bias_ih_l%d' % l] = u(3 * H); w['bias_hh_l%d' % l] = u(3 * H)
  return w


def bits(a):
  return np.asarray(a, np.float32).view(np.uint32)


def device_score(m, xs, labels, frames=True, stream=None):
  """uis_score_device on fp32 copies of xs / labels: (scores [U], list of per-frame increments or None)."""
  import torch
  off = np.concatenate([[0], np.cumsum([len(x) for x in xs])]).astype(np.int64)
  x_dev = torch.from_numpy(np.concatenate([np.asarray(x, np.float32).reshape(-1, m.D) for x in xs])).cuda()
  l_dev = torch.from_numpy(np.concatenate([np.asarray(l, np.int32) for l in labels])).cuda()
  s_dev = torch.full((len(xs),), np.nan, dtype=torch.float32, device='cuda')
  f_dev = torch.full((max(int(off[-1]), 1),), np.nan, dtype=torch.float32, device='cuda')
  torch.cuda.synchronize()
  if stream is None:
    m.score_device(x_dev.data_ptr(), off, l_dev.data_ptr(), s_dev.data_ptr(), f_dev.data_ptr() if frames else 0)
    torch.cuda.synchronize()
  else:
    with torch.cuda.stream(stream):
      m.score_device(x_dev.data_ptr(), off, l_dev.data_ptr(), s_dev.data_ptr(), f_dev.data_ptr() if frames else 0,
                     stream=stream.cuda_stream)
    stream.synchronize()
  f = f_dev.cpu().numpy()
  return s_dev.cpu().numpy(), [f[off[u]:off[u + 1]] for u in range(len(xs))] if frames else None


def check_frames(key, scores, frames, inc, gauss):
  """Per frame within the allowance of the float64 rescore (inc, gauss: lists per utterance); every total the bits of
  the fp32 running sum of its frames."""
  for u, (s, f, i, g) in enumerate(zip(scores, frames, inc, gauss)):
    assert f.dtype == np.float32 and len(f) == len(i)
    share = frame_share(f, i, g)
    assert np.all(share <= 1), (key, u, int(np.argmax(share)), float(share.max()), float(f[np.argmax(share)]),
                                float(i[np.argmax(share)]))
    note(key, float(share.max(initial=0)))
    assert bits(s) == bits(fp32_sum(f)), (key, u, float(s), float(fp32_sum(f)))


def rescore(w, xs, labels, mean0=None):
  ps = path_score(w, xs, [np.asarray(l)[None] for l in labels], mean0=mean0, device='cuda', per_frame=True)
  return ps.frame_inc, ps.frame_gauss


def both_entry_points(m, w, xs, labels, key, mean0=None, rescored=None):
  """Host and device entry points, bit-equal to each other and per frame within the rescore's allowance."""
  got, frames = m.score(xs, labels, per_frame=True)
  dg, dframes = device_score(m, xs, labels)
  assert np.array_equal(bits(got), bits(dg))
  assert all(np.array_equal(bits(a), bits(b)) for a, b in zip(frames, dframes))
  inc, gauss = rescored or rescore(w, xs, labels, mean0)
  check_frames(key, got, frames, inc, gauss)
  return got, frames


# ---- the reference's golden cases

_GOLDEN = {}


def golden_rescore(model_name):
  """{case name: (increments, Gaussian terms)} of one model's golden cases, one batched rescore on the GPU."""
  if model_name not in _GOLDEN:
    cases = [c for c in CASES if c['model'] == model_name]
    inc, gauss = rescore(load_weights(model_name), [c['x'] for c in cases], [c['labels'] for c in cases])
    _GOLDEN[model_name] = {c['name']: (i, g) for c, i, g in zip(cases, inc, gauss)}
  return _GOLDEN[model_name]


@pytest.mark.parametrize('model_name', sorted({c['model'] for c in CASES}))
def test_golden_cases_per_frame(native, model_name):
  """Every golden case through both entry points: per frame within the rescore's allowance, within twice of it of the
  reference's own per-frame losses (each lies within one), and totals within the rescore's total allowance."""
  cases = [c for c in CASES if c['model'] == model_name]
  w = load_weights(model_name)
  m = native.NativeModel(w)
  xs, labels = [c['x'] for c in cases], [c['labels'] for c in cases]
  r = golden_rescore(model_name)
  inc, gauss = [r[c['name']][0] for c in cases], [r[c['name']][1] for c in cases]
  got, frames = both_entry_points(m, w, xs, labels, 'golden ' + model_name, rescored=(inc, gauss))
  same = 0
  for c, f, i, g in zip(cases, frames, inc, gauss):
    assert np.all(np.abs(f.astype(np.float64) - c['frames']) <= 2 * frame_allowance(i, g)), c['name']
    same += int(np.sum(bits(f) == bits(c['frames'])))
  note('golden %s frames = reference' % model_name, '%d / %d' % (same, sum(len(f) for f in frames)))
  ps = path_score(w, xs, [l[None] for l in labels], device='cuda')
  assert np.all(ps.share(got) <= 1)


# ---- kernel shapes, depths, zero-padded shapes

@pytest.mark.parametrize('H,D,depth', SHAPES + PADDED)
def test_kernel_shapes_per_frame(native, H, D, depth):
  w = large_model(H, D, depth, seed=7000 + H + D + depth) if (H, D, depth) in SHAPES else padded_model(H, D, depth)
  m = native.NativeModel(w)
  rng = np.random.default_rng(H + D + depth)
  xs = utterances(D, 7800 + depth, (37, 1, 60, 0, 23))
  labels = [random_labels(rng, len(x), k) for x, k in zip(xs, (5, 1, 9, 1, 23))]
  mean0, _ = m.constants()
  both_entry_points(m, w, xs, labels, 'shape %dx%d d%d' % (H, D, depth), mean0=mean0)
  assert m.stats()['engine'] == 1


# ---- the reduce kernel's log tables past 4096 entries; thousands of clusters

def test_turns_past_4096_grow_the_log_tables_from_score(native):
  """s_alternating: 4399 turns, read at index 4399 of the ddCRP denominator's table.  A fresh handle grows its tables
  from the score call itself; a second handle first decodes a short utterance (tables at their default 4096 entries)
  and then grows them from the score call.  Both give the same bits."""
  c = next(c for c in CASES if c['name'] == 's_alternating')
  w = load_weights(c['model'])
  inc, gauss = golden_rescore(c['model'])[c['name']]
  fresh = native.NativeModel(w)
  got, frames = fresh.score([c['x']], [c['labels']], per_frame=True)
  check_frames('turns > 4096', got, frames, [inc], [gauss])
  after = native.NativeModel(w)
  assert len(after.predict([c['x'][:40]], beam_size=4, test_iteration=1)[0]) == 40
  got2, frames2 = both_entry_points(after, w, [c['x']], [c['labels']], 'turns > 4096', rescored=([inc], [gauss]))
  assert bits(got2) == bits(got) and np.array_equal(bits(frames2[0]), bits(frames[0]))


def test_3000_clusters_in_one_utterance(native):
  c = next(c for c in CASES if c['name'] == 's_3000_clusters')
  w = load_weights(c['model'])
  m = native.NativeModel(w)
  both_entry_points(m, w, [c['x']], [c['labels']], '3000 clusters', rescored=tuple(
      [v] for v in golden_rescore(c['model'])[c['name']]))
  st = m.stats()
  assert st['max_k'] == 3000
  assert st['gru_columns'] == len(c['labels']) - 3000


# ---- edges of the chain plan

SMALL = 'model_small.npz'


def small(native):
  w = load_weights(SMALL)
  return w, native.NativeModel(w)


def test_no_chain_queued_skips_the_chain_kernel(native):
  """Every chain one frame long: nothing is queued and the chain kernel is not launched (first-visit and reduce
  kernels only, after the device entry point's input projection)."""
  w, m = small(native)
  xs = utterances(64, 7500, (30, 1, 12, 0))
  labels = [np.arange(len(x), dtype=np.int32) for x in xs]
  inc, gauss = rescore(w, xs, labels)
  got, frames = m.score(xs, labels, per_frame=True)
  st = m.stats()
  assert st['ctas'] == 0 and st['gru_columns'] == 0 and st['weight_passes'] == 0
  assert st['kernel_launches'] == 2 + 2 * st['chunks']
  dg, dframes = device_score(m, xs, labels)
  st = m.stats()
  assert st['ctas'] == 0 and st['gru_columns'] == 0 and st['kernel_launches'] == 3
  assert np.array_equal(bits(got), bits(dg)) and all(np.array_equal(bits(a), bits(b)) for a, b in zip(frames, dframes))
  check_frames('chain plan', got, frames, inc, gauss)


def test_exactly_one_queued_chain(native):
  w, m = small(native)
  xs = utterances(64, 7510, (9, 14))
  labels = [np.array([0, 1, 2, 0, 3, 4, 0, 5, 0], np.int32), np.arange(14, dtype=np.int32)]
  both_entry_points(m, w, xs, labels, 'chain plan')
  st = m.stats()
  assert st['ctas'] == 1 and st['gru_columns'] == 3 and st['weight_passes'] == 3


def test_chains_of_two_frames_take_one_pass_and_retire(native):
  """Every chain two frames long: each column takes one pass and hands on, and the queue runs out mid-CTA."""
  w, m = small(native)
  rng = np.random.default_rng(7520)
  from uisrnn_b200.uisrnn import canonical_labels
  xs = utterances(64, 7520, (40, 18, 64))
  labels = [canonical_labels(rng.permutation(np.arange(len(x)) // 2)) for x in xs]
  both_entry_points(m, w, xs, labels, 'chain plan')
  st = m.stats()
  queued = sum(len(x) // 2 for x in xs)
  assert st['gru_columns'] == queued and st['ctas'] == (queued + 19) // 20  # 20 columns per CTA (beam_cp)


def test_more_chains_than_resident_columns_refill(native):
  """More queued chains than SMs x columns per CTA (20 at hidden <= 512: beam_cp in uis_beam.cuh): every CTA
  refills columns from the queue while others still run."""
  import torch
  w, m = small(native)
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  n_utt = sms * 20 // 10 + 60
  rng = np.random.default_rng(7530)
  from uisrnn_b200.uisrnn import canonical_labels
  xs = utterances(64, 7530, (30,) * n_utt)
  labels = [canonical_labels(rng.permutation(np.arange(30) % 10)) for _ in xs]
  assert 10 * n_utt > sms * 20
  both_entry_points(m, w, xs, labels, 'chain plan')
  st = m.stats()
  assert st['ctas'] == sms and st['gru_columns'] == 20 * n_utt
  assert st['weight_passes'] > 2 * sms  # two passes per chain, more chains than columns


def test_first_column_rule_on_a_new_cluster(native):
  """A frame whose x[0] equals the kernel's fp32 mean0[0] and that opens a new cluster scores +inf; the total is
  +inf and every later frame stays finite (the cluster's state still advances)."""
  w, m = small(native)
  mean0, _ = m.constants()
  rng = np.random.default_rng(7540)
  x = utterances(64, 7540, (40,))[0].copy()
  lab = random_labels(rng, 40, 4)
  t = int(np.nonzero(lab == 2)[0][0])
  assert t > 0
  x[t, 0] = float(np.float32(mean0[0]))
  got, frames = both_entry_points(m, w, [x], [lab], 'first-column rule', mean0=mean0)
  f = frames[0]
  assert np.isinf(got[0]) and np.isinf(f[t]) and np.all(np.isfinite(np.delete(f, t)))


# ---- entry points

def golden_small():
  cases = [c for c in CASES if c['model'] == SMALL and len(c['x']) < 1000]
  return [c['x'] for c in cases], [c['labels'] for c in cases]


def test_device_entry_without_frames_and_on_a_side_stream(native):
  import torch
  w, m = small(native)
  xs, labels = golden_small()
  got, frames = m.score(xs, labels, per_frame=True)
  s0, none = device_score(m, xs, labels, frames=False)
  assert none is None and np.array_equal(bits(s0), bits(got))
  side = torch.cuda.Stream()
  s1, f1 = device_score(m, xs, labels, stream=side)
  assert np.array_equal(bits(s1), bits(got)) and all(np.array_equal(bits(a), bits(b)) for a, b in zip(f1, frames))


def test_device_entry_rejects_non_canonical_labels(native):
  w, m = small(native)
  xs, labels = golden_small()
  bad = [np.asarray(l, np.int32).copy() for l in labels]
  bad[1][5] = bad[1][:5].max() + 2
  with pytest.raises(native.NativeError) as err:
    device_score(m, xs, bad)
  assert err.value.code == native.UIS_ERR_INVALID
  assert 'utterance 1 frame 5' in str(err.value)


@pytest.mark.parametrize('staging', ['0', '1'])
def test_host_staging_chunks_give_the_same_bits(native, monkeypatch, staging):
  """256-row staging chunks (UISRNN_B200_CHUNK_MB=0), with and without the pinned staging ring: chunk boundaries fall
  inside utterances and inside chains; the result is the default call's, bit for bit."""
  w, m = small(native)
  rng = np.random.default_rng(7550)
  xs = utterances(64, 7550, (300, 500, 41))
  labels = [random_labels(rng, len(x), 7) for x in xs]
  got, frames = both_entry_points(m, w, xs, labels, 'host staging')
  monkeypatch.setenv('UISRNN_B200_CHUNK_MB', '0')
  monkeypatch.setenv('UISRNN_B200_HOST_STAGING', staging)
  g2, f2 = m.score(xs, labels, per_frame=True)
  st = m.stats()
  assert st['chunks'] >= 4 and st['staged'] == int(staging)
  assert np.array_equal(bits(g2), bits(got)) and all(np.array_equal(bits(a), bits(b)) for a, b in zip(f2, frames))


# ---- N-best scores of the beam kernels against score()

def nbest_seqs(m, xs, k, **kw):
  """predict(n_best=k) at test_iteration 1: (inputs, labels, scores) of every returned hypothesis."""
  labels, scores, _, count = m.predict(xs, test_iteration=1, n_best=k, **kw)
  seqs = [x for u, x in enumerate(xs) for _ in range(count[u])]
  labs = [labels[u][j] for u in range(len(xs)) for j in range(count[u])]
  want = np.array([scores[u][j] for u in range(len(xs)) for j in range(count[u])], np.float32)
  return seqs, labs, want


def toy_utts(n, seed):
  from uisrnn_b200.synth import synth_utt
  return [synth_utt(seed + u, n_frames=40 + 11 * u, n_spk=4, noise=0.06)[0] for u in range(n)]


NBEST = {
    '1024x512-d1': lambda nat: (_cached(nat, 1024, 512, 1)[1], utterances(512, 7600, (26, 33)), 5, dict(beam_size=5)),
    '1024x512-d2': lambda nat: (_cached(nat, 1024, 512, 2)[1], utterances(512, 7610, (26, 33)), 5, dict(beam_size=5)),
    '256x128-d3': lambda nat: (_cached(nat, 256, 128, 3)[1], utterances(128, 7620, (30, 45)), 6, dict(beam_size=8)),
    '256x128-d4': lambda nat: (_cached(nat, 256, 128, 4)[1], utterances(128, 7630, (30, 45)), 6, dict(beam_size=8)),
    'padded-600x300': lambda nat: (_cached(nat, 600, 300, 1)[1], utterances(300, 7640, (26, 33)), 5,
                                   dict(beam_size=5)),
    'toy-beam64': lambda nat: (nat.NativeModel(load_weights('model_toy100.npz')), toy_utts(2, 7650), 64,
                               dict(beam_size=64, max_speakers=4)),
    'toy-beam128': lambda nat: (nat.NativeModel(load_weights('model_toy100.npz')), toy_utts(1, 7660), 128,
                                dict(beam_size=128, max_speakers=4)),
    'toy-lanes2': lambda nat: (nat.NativeModel(load_weights('model_toy100.npz')), toy_utts(5, 7670), 10,
                               dict(beam_size=10, lanes=2)),
}


@pytest.mark.parametrize('variant', list(NBEST))
def test_ffma_nbest_scores_are_score_bits(native, variant):
  """A hypothesis the FFMA beam kernel kept scores, through score(), exactly its N-best score: the two share the
  weight pass and the Gaussian term (DESIGN section 4.1)."""
  m, xs, k, kw = NBEST[variant](native)
  seqs, labs, want = nbest_seqs(m, xs, k, look_ahead=1, engine=1, cluster=-1, **kw)
  assert m.stats()['engine'] == 1 and len(want) >= min(k, 2) * len(xs) // 2 and np.all(np.isfinite(want))
  got = m.score(seqs, labs)
  assert np.array_equal(bits(got), bits(want)), int(np.argmax(bits(got) != bits(want)))


@pytest.mark.parametrize('spill', [False, True])
def test_tree_nbest_within_the_rescore(native, monkeypatch, spill):
  """The look_ahead-2 tree kernel (shared memory, and spilled to its device arena) scores its own sub-steps: its
  N-best scores lie within the total allowance of the float64 rescore, and so do score()'s of the same labels.
  Whether the bits agree is recorded, not required."""
  if spill:
    monkeypatch.setenv('UISRNN_B200_TREE_SPILL', 'force')
  w = load_weights('model_toy100.npz')
  m = native.NativeModel(w)
  xs = toy_utts(3, 7680)
  seqs, labs, want = nbest_seqs(m, xs, 5, beam_size=10, look_ahead=2)
  got = m.score(seqs, labs)
  ps = path_score(w, seqs, [np.asarray(l)[None] for l in labs], device='cuda')
  assert np.all(ps.share(want) <= 1) and np.all(ps.share(got) <= 1)
  note('tree%s N-best = score() bits' % (' spilled' if spill else ''),
       '%d / %d' % (int(np.sum(bits(got) == bits(want))), len(want)))
