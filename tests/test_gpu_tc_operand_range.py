"""The tensor-core weight pass pinned per beam step to the float64 replay at the edges of its fp16 operand scales.

tc_prepare (uisrnn_b200/csrc/uis_api.cu) picks one power of two per operand so that v * 2^s = hi + lo in two fp16
halves: one per weight matrix from its max |w|, one for the hidden columns from max(1, max |hidden0|) and one for
a = relu(W1 h' + b1) from the bound max_i |b1_i| + hmax * sum_j |W1_ij|.  The models of tests/test_gpu_step_replay.py
keep every bound a few bits above the values it scales.  Here each case moves one scale to an edge while the means stay
O(1) and informative: a loose bound on a (large b1 or a large, cancelling W1 row on a unit whose W2 column is zero), a
loose bound on h (large rnn_init_hidden on units no product reads), one weight far above its matrix's others, the
whole W2 operand x 2^+-12 and 2^+-24 (the clamp of tc_pow2_scale binds at 2^-24), max |w| and max |hidden0| exactly at a
power of two and one fp32 ulp above, and models whose scales leave the engine no planes (the FFMA kernels serve them).

Every case decodes frames clustered around the model's own mean0 on the tensor-core engine and checks each beam step
with tests/beam_replay.py at its unchanged INC_RTOL / STATE_TOL, and replays the same model once on the FFMA engine as
a control.  Every call asserts the engine that ran.  The worst share of the allowance per case is printed (-s)."""

import numpy as np
import pytest

import beam_replay as R

pytestmark = pytest.mark.gpu

INC_RTOL, STATE_TOL = R.INC_RTOL, R.STATE_TOL
WORST = {}  # (case id, engine) -> {'inc' | 'mean' | 'hidden': worst share of the allowance}


@pytest.fixture(scope='module')
def native():
  from uisrnn_b200 import native as nat
  nat.load_library()
  return nat


def random_weights(H, D, seed):
  """An untrained depth-1 model with small recurrent weights (test_gpu_step_replay.random_weights)."""
  rng = np.random.default_rng(seed)
  u = lambda *s: (rng.uniform(-1, 1, size=s) / np.sqrt(H)).astype(np.float32)
  return {'depth': 1, 'w1': u(H, H), 'b1': u(H), 'w2': u(D, H), 'b2': u(D), 'h0': u(1, 1, H),
          'sigma2': (0.05 + 0.1 * rng.random(D)).astype(np.float32), 'transition_bias': 0.15, 'crp_alpha': 1.0,
          'weight_ih_l0': u(3 * H, D), 'weight_hh_l0': u(3 * H, H), 'bias_ih_l0': u(3 * H), 'bias_hh_l0': u(3 * H)}


def clustered(rng, n, D, spk=3, run=7, scale=0.3, noise=0.05):
  centres = rng.standard_normal((spk, D))
  return centres[(np.arange(n) // run) % spk] * scale + noise * rng.standard_normal((n, D))


MATRIX = {'whh': 'weight_hh_l0', 'w1': 'w1', 'w2': 'w2'}


def loose_amax(b1):
  def edit(w):
    w['b1'][3] = b1
    w['w2'][:, 3] = 0  # a_3 ~ b1 reaches no mean
  return edit


def cancelling_w1_row(w):
  """Row 3 of W1 alternates +-c, sum |W1_3j| = 1e6: the bound on a grows by ~2^20, W1 h on that row stays ~1e4."""
  H = w['w1'].shape[1]
  w['w1'][3] = np.float32(1e6 / H) * np.where(np.arange(H) % 2, -1, 1).astype(np.float32)
  w['w2'][:, 3] = 0


def loose_hmax(h):
  def edit(w):
    units = [5, 6, 7]
    w['h0'][0, 0, units] = np.float32(h) * np.array([1, -1, 0.5], np.float32)
    w['weight_hh_l0'][:, units] = 0  # no gate reads them
    w['w1'][:, units] = 0            # nor W1: the means stay O(1)
  return edit


def outlier(mat, log2f):
  """One entry of a matrix 2^log2f times its largest; W1 row 3 / W2 column 3 cut from the means."""
  def edit(w):
    a = w[MATRIX[mat]]
    a[3, 5] = np.float32(np.abs(a).max() * 2.0 ** log2f)
    if mat == 'w1':
      w['w2'][:, 3] = 0        # a_3 is large
    elif mat == 'w2':
      w['w1'][5] = 0           # a_5 = relu(0 - 1) = 0: the outlier multiplies zero
      w['b1'][5] = -1
  return edit


def operand_scale(log2f):
  """W2, b2 (and the frames) x f, W_ih x 1 / f (the GRU sees the same input), sigma2 x f^2 (same Gaussian terms)."""
  def edit(w):
    f = np.float32(2.0 ** log2f)
    w['w2'] *= f
    w['b2'] *= f
    w['weight_ih_l0'] /= f
    w['sigma2'] *= f * f
  return edit, 2.0 ** log2f


def pow2_max(above):
  """max |w| of W_hh, W1 and W2 exactly 2^-4 (their scale puts it at 2^14), or one fp32 ulp above."""
  def edit(w):
    v = np.float32(2.0 ** -4)
    if above:
      v = np.nextafter(v, np.float32(1))
    for k, mat in enumerate(MATRIX.values()):
      w[mat][3 + k, 5] = -v if k == 1 else v
    w['w1'][5] = 0  # a_5 = 0 under the W2 entry
    w['b1'][5] = -1
  return edit


def unit_hidden0(above):
  """hidden0_9 = h0_9 exactly (n_9 = tanh(0) = 0, z_9 = 1 in fp32): max |hidden0| is 1, or one fp32 ulp above it."""
  def edit(w):
    H = w['w1'].shape[0]
    w['h0'][0, 0, 9] = np.nextafter(np.float32(1), np.float32(2)) if above else np.float32(1)
    for k in ('weight_ih_l0', 'weight_hh_l0', 'bias_ih_l0', 'bias_hh_l0'):
      w[k][2 * H + 9] = 0
    w['bias_hh_l0'][H + 9] = 60.0
  return edit, 1.0, (np.nextafter(np.float32(1), np.float32(2)) if above else np.float32(1))


# case id -> (edit, frame scale, expected max |hidden0| or None); the tensor-core engine serves every one of them
CASES = {
    'amax_b1_1e4': (loose_amax(1e4), 1.0, None),
    'amax_b1_1e5': (loose_amax(1e5), 1.0, None),
    'amax_b1_1e6': (loose_amax(1e6), 1.0, None),
    'amax_w1_cancelling': (cancelling_w1_row, 1.0, None),
    'hmax_1e3': (loose_hmax(1e3), 1.0, None),
    'hmax_1e5': (loose_hmax(1e5), 1.0, None),
    'whh_outlier_2^10': (outlier('whh', 10), 1.0, None),
    'whh_outlier_2^17': (outlier('whh', 17), 1.0, None),
    'w1_outlier_2^10': (outlier('w1', 10), 1.0, None),
    'w1_outlier_2^17': (outlier('w1', 17), 1.0, None),
    'w2_outlier_2^10': (outlier('w2', 10), 1.0, None),
    'w2_outlier_2^17': (outlier('w2', 17), 1.0, None),
    'w2_x2^12': operand_scale(12) + (None,),
    'w2_x2^-12': operand_scale(-12) + (None,),
    'w2_x2^24': operand_scale(24) + (None,),
    'w2_x2^-24': operand_scale(-24) + (None,),
    'max_w_pow2': (pow2_max(False), 1.0, None),
    'max_w_pow2_ulp_above': (pow2_max(True), 1.0, None),
    'hidden0_one': unit_hidden0(False),
    'hidden0_one_ulp_above': unit_hidden0(True),
}
# split too lossy (tc_prepare's kTcSplitLoss): the FFMA engine serves these models
FALLBACK_OUTLIERS = {'whh_outlier_2^24': outlier('whh', 24), 'w1_outlier_2^24': outlier('w1', 24),
                     'w2_outlier_2^24': outlier('w2', 24)}
PADDED = ['amax_b1_1e6', 'amax_w1_cancelling', 'hmax_1e5', 'w1_outlier_2^17', 'w2_x2^-24', 'max_w_pow2_ulp_above']

TC_KW = dict(engine=2, lanes=2, n_ctas=1)
TC_STATS = dict(engine=2, lanes=2, tc_columns=48, cluster=1, ctas=1)
FFMA_KW = dict(engine=1, lanes=1, cluster=-1, n_ctas=2)
FFMA_STATS = dict(engine=1, lanes=1, tc_columns=0, cluster=1, ctas=2)


def build(native, H, D, edit, seed):
  w = random_weights(H, D, seed)
  edit(w)
  nm = native.NativeModel(w)
  return w, nm, R.Model(w)


def inputs(rm, seed, scale=1.0):
  """Two utterances (31, 18 frames) clustered around the model's own mean0, their spread x the case's frame scale."""
  rng = np.random.default_rng(seed)
  return [rm.mean0 + scale * clustered(rng, n, rm.D) for n in (31, 18)]


def replay(case, nm, rm, xs, kw, expect):
  """Decodes xs once per utterance with its trace and checks each against the replay; records the worst shares."""
  mean0 = nm.constants()[0]
  worst = {}
  for u in range(len(xs)):
    labels, dbg = nm.predict(xs, trace_utt=u, **kw)
    st = nm.stats()
    got = {k: st[k] for k in expect}
    assert got == expect, '%s utterance %d ran %s, expected %s' % (case, u, got, expect)
    rp = R.Replay(rm, xs[u], 10, 1, 2, dbg['win'], dbg['score'], dbg['off'], mean0=mean0)
    final = dict(best_mean=dbg['best_mean'], best_hidden=dbg['best_hidden'], best_blocks=dbg['best_blocks'],
                 final_k=dbg['final_k'][u], final_scores=dbg['final_scores'][u])
    try:
      R.check(rp, INC_RTOL, labels=labels[u].tolist(), final=final, state_tol=STATE_TOL, worst=worst)
    finally:
      share = {'inc': worst.get('inc', 0.0) / INC_RTOL, 'mean': worst.get('mean', 0.0) / STATE_TOL,
               'hidden': worst.get('hidden', 0.0) / STATE_TOL}
      WORST[(case, expect['engine'])] = share
      print(' %s engine %d worst share: %s' % (case, expect['engine'],
                                              ', '.join('%s %.3f' % kv for kv in sorted(share.items()))), end='')


def auto_engine(nm, xs):
  """The engine the automatic plan takes for two utterances on one CTA (the tensor cores whenever the model has planes)."""
  nm.predict(xs, n_ctas=1)
  return nm.stats()['engine']


@pytest.mark.parametrize('H,D', [(512, 256), (300, 200), (256, 128)])
@pytest.mark.parametrize('case', list(CASES))
def test_tensor_cores_at_operand_scale_edges(native, case, H, D):
  if (H, D) != (512, 256) and case not in PADDED:
    pytest.skip('zero-padded shapes run a subset')
  edit, fscale, hidden0_max = CASES[case]
  seed = 7000 + list(CASES).index(case) + 100 * (H // 128)
  _, nm, rm = build(native, H, D, edit, seed)
  if hidden0_max is not None:  # the boundary is where the case means it to be
    assert np.max(np.abs(nm.constants()[1])) == hidden0_max
  xs = inputs(rm, seed, fscale)
  assert auto_engine(nm, xs) == 2
  replay(case + '@%dx%d' % (H, D), nm, rm, xs, TC_KW, TC_STATS)
  replay(case + '@%dx%d' % (H, D), nm, rm, xs, FFMA_KW, FFMA_STATS)


def fallback_models():
  out = dict(FALLBACK_OUTLIERS)

  def zero_w2(w):
    w['w2'][:] = 0

  def clamped_amax(w):  # bound ~1e17 > 2^54: tc_pow2_scale returns 0 for a
    loose_amax(1e17)(w)
  out['w2_zero'] = zero_w2
  out['amax_clamps_to_zero'] = clamped_amax
  return out


FALLBACK = fallback_models()


@pytest.mark.parametrize('case', list(FALLBACK))
def test_models_without_planes_decode_on_ffma(native, case):
  """Under the automatic plan these models decode on the FFMA engine, bit for bit as a forced engine=1 call; a forced
  engine=2 call is refused (the tensor-core kernel never runs without planes).  The decode replays within bounds."""
  seed = 7500 + list(FALLBACK).index(case)
  _, nm, rm = build(native, 512, 256, FALLBACK[case], seed)
  xs = inputs(rm, seed)
  assert auto_engine(nm, xs) == 1
  auto = nm.predict(xs, n_ctas=1, n_best=3)
  assert nm.stats()['engine'] == 1
  ffma = nm.predict(xs, n_ctas=1, n_best=3, engine=1)
  for a, b in zip(auto[0], ffma[0]):
    assert np.array_equal(a, b)
  assert np.array_equal(auto[1].view(np.uint32), ffma[1].view(np.uint32))
  with pytest.raises(native.NativeError, match='tensor-core engine'):
    nm.predict(xs, n_ctas=1, engine=2)
  replay(case, nm, rm, xs, FFMA_KW, FFMA_STATS)


def test_report_worst():
  """Runs last in this file: the worst share of the allowance per case and engine (shown with -s)."""
  print('\nkernel vs float64 replay, worst share of the allowance (inc, mean, hidden) per case:')
  for (case, engine), s in sorted(WORST.items()):
    print('  %-36s engine %d  inc %.3f  mean %.3f  hidden %.3f' % (case, engine, s['inc'], s['mean'], s['hidden']))
  assert all(v <= 1.0 for s in WORST.values() for v in s.values())
