"""Pins EVERY kernel variant of the look_ahead-1 beam search -- in particular the one `bench.py` times (lanes = 2,
one CTA per lane group, no cluster) -- to labels produced by the unmodified reference at the full length of the
benchmark utterances (500 frames = 1000 beam steps: slot recycling, queue refill), and to the CPU oracle on the other
kernel shapes.  VERDICT round 1, "What's weak" item 1.

Variants are forced through the C ABI's `lanes` / `cluster` options (`include/uisrnn_b200.h`, uis_predict_opts):
  lanes=2 cluster=-1   uis_beam_kernel<H,D,false,false>, two utterances per CTA sharing each weight pass (bench path)
  lanes=1 cluster=-1   the same kernel, one utterance per CTA
  lanes=0 cluster=0    automatic choice (few utterances -> thread-block-cluster kernel)
  lanes=0 cluster=32   stationary-weights mode (groups of 32 CTAs, weights resident in shared memory)
  engine=2             the tensor-core pass (wgmma): tests/test_gpu_tensorcore.py
"""
import numpy as np
import pytest

from helpers import GOLDEN, load_weights, uis_oracle

pytestmark = pytest.mark.gpu

VARIANTS = [dict(lanes=2, cluster=-1, engine=1), dict(lanes=1, cluster=-1, engine=1), dict(lanes=0, cluster=0, engine=1),
            dict(lanes=4, cluster=-1, engine=1), dict(lanes=0, cluster=32, engine=0)]


@pytest.fixture(scope='module')
def native():
  from uisrnn_b200 import native as nat
  nat.load_library()
  return nat


@pytest.fixture(scope='module')
def toy_model(native):
  return native.NativeModel(load_weights('model_toy100.npz'))


@pytest.fixture(scope='module')
def small_model(native):
  return native.NativeModel(load_weights('model_small.npz'))


def _bench_golden():
  from uisrnn_b200.synth import synth_utt
  g = np.load(GOLDEN + '/synth500_bench.npz')
  xs = [synth_utt(int(s))[0] for s in g['seeds']]
  return [int(s) for s in g['seeds']], xs, [lab.tolist() for lab in g['labels']]


@pytest.mark.parametrize('opts', VARIANTS, ids=lambda o: 'lanes%d_cluster%d' % (o['lanes'], o['cluster']))
def test_default_shape_500_frames_reference_labels(toy_model, opts):
  """(hidden, dim) = (512, 256): ten utterances of bench.py's workload + the two of synth500.npz, 1000 beam steps."""
  from uisrnn_b200.synth import synth_utt
  _, xs, want = _bench_golden()
  g2 = np.load(GOLDEN + '/synth500.npz')
  xs = xs + [synth_utt(int(s))[0] for s in g2['seeds']]
  want = want + [lab.tolist() for lab in g2['labels']]
  got = toy_model.predict(xs, **opts)
  st = toy_model.stats()
  if opts['lanes'] in (1, 2):
    assert st['lanes'] == opts['lanes'] and st['cluster'] == 1
  for i, (g, w) in enumerate(zip(got, want)):
    assert g.tolist() == w, 'utterance %d, variant %r' % (i, opts)


@pytest.mark.parametrize('opts', VARIANTS[:2], ids=lambda o: 'lanes%d' % o['lanes'])
def test_small_shape_500_frames_reference_labels(small_model, opts):
  """(128, 64): four 500-frame utterances decoded by the reference (tests/golden/small500.npz)."""
  from uisrnn_b200.synth import synth_utt
  g = np.load(GOLDEN + '/small500.npz')
  xs = [synth_utt(int(s), n_frames=500, dim=64, n_spk=4, noise=0.08)[0] for s in g['seeds']]
  got = small_model.predict(xs, **opts)
  assert small_model.stats()['lanes'] == opts['lanes']
  for o, w in zip(got, g['labels']):
    assert o.tolist() == w.tolist()


def _random_weights(H, D, seed):
  rng = np.random.default_rng(seed)
  u = lambda *s: (rng.uniform(-1, 1, size=s) / np.sqrt(H)).astype(np.float32)
  return {'depth': 1, 'weight_ih_l0': u(3 * H, D), 'weight_hh_l0': u(3 * H, H), 'bias_ih_l0': u(3 * H),
          'bias_hh_l0': u(3 * H), 'w1': u(H, H), 'b1': u(H), 'w2': u(D, H), 'b2': u(D),
          'h0': u(1, 1, H), 'sigma2': (0.05 + 0.1 * rng.random(D)).astype(np.float32),
          'transition_bias': 0.1, 'crp_alpha': 1.0}


@pytest.mark.parametrize('opts', VARIANTS[:2], ids=lambda o: 'lanes%d' % o['lanes'])
def test_mid_shape_matches_oracle(native, opts):
  """(256, 128) has no reference-trained fixture: untrained weights against the oracle, 6 utterances x 120 frames."""
  H, D = 256, 128
  w = _random_weights(H, D, 11)
  model = native.NativeModel(w)
  om = uis_oracle.OracleModel(w)
  rng = np.random.default_rng(5)
  centres = rng.standard_normal((3, D))
  xs = []
  for n in (120, 97, 120, 64, 120, 33):
    lab = (np.arange(n) // 11) % 3
    xs.append(centres[lab] * 0.3 + 0.05 * rng.standard_normal((n, D)))
  got = model.predict(xs, kcap=64, **opts)
  assert model.stats()['lanes'] == opts['lanes']
  for x, o in zip(xs, got):
    assert o.tolist() == uis_oracle.predict_single(om, x, beam_size=10, look_ahead=1, test_iteration=2)


def test_full_bench_batch_first_median_last(toy_model):
  """One call with bench.py's whole per-GPU batch (296 utterances x 500 frames, automatic options = what the bench
  launched in round 1 -- the FFMA engine with two lanes): the utterances the reference decoded (first six, median two, last two) must come out identical, and
  the device-resident entry point must agree with the host entry point on every utterance."""
  import torch
  from uisrnn_b200.synth import synth_utt
  seeds, _, want = _bench_golden()
  U = 296
  xs = [synth_utt(100000 + u)[0] for u in range(U)]
  got = toy_model.predict(xs, engine=1)
  st = toy_model.stats()
  assert st['lanes'] == 2 and st['cluster'] == 1 and st['utterances'] == U and st['engine'] == 1
  for s, w in zip(seeds, want):
    assert got[s - 100000].tolist() == w, 'utterance %d of the bench batch' % (s - 100000)
  x_dev = torch.from_numpy(np.concatenate(xs).astype(np.float32)).cuda()
  lab_dev = torch.empty(U * 500, dtype=torch.int32, device='cuda')
  toy_model.predict_device(x_dev.data_ptr(), np.arange(U + 1, dtype=np.int64) * 500, lab_dev.data_ptr(), engine=1)
  assert np.array_equal(lab_dev.cpu().numpy(), np.concatenate(got))
