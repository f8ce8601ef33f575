"""Every predict() kernel pinned per beam step to a float64 replay of its own trace (tests/beam_replay.py).

The parity tests compare cumulative scores within 1e-5 of the score, which allows a larger error in each step's
increment as a decode goes on (about 0.2 % of one increment after the toy trace's 190 steps, about 4 % after 4000).
Here each traced step is checked on its own: from the kernel's own previous scores, every winner's increment against
the float64 increment (one fp32 ulp of the score per sub-step + INC_RTOL of the increment), the selection (winner count
min(#finite, B), no loser below a winner, ranks in order, all up to that tolerance), the rank-0 state at the end (each
cluster's mean row and each (cluster, layer) hidden row against its own scale; blocks and K exact; final scores equal
to the last step's) and the labels (the back-track of the trace from the rank the min_speakers rule picks).  Every call
also asserts which kernel ran (stats: engine, lanes, tensor-core columns, cluster, CTAs), so a silent fall-back to
another kernel fails.

The matrix traces every lane of CTAs that hold several, both engines, the cluster and stationary-weights modes, depth
1-4, zero-padded shapes, the look-ahead tree kernel in shared memory and spilled, speaker bounds, host staging chunks,
edge inputs and 4200-step decodes (beyond the 4094 steps the default log tables hold).  What stays unchecked here:
predict_device (it takes no taps), utterances that are not traced in a call (their labels only) and calls on every SM;
tests/test_gpu_full_occupancy.py covers those."""

import numpy as np
import pytest

import beam_replay as R
from helpers import load_weights

pytestmark = pytest.mark.gpu

INC_RTOL, STATE_TOL = R.INC_RTOL, R.STATE_TOL  # (measured worst beside them in beam_replay.py)
# worst error seen per class in this session (what the bounds above were calibrated from)
WORST = {}


@pytest.fixture(scope='module')
def native():
  from uisrnn_b200 import native as nat
  nat.load_library()
  return nat


def random_weights(H, D, depth=1, seed=0, p0=0.15, alpha=1.0):
  """An untrained model: small recurrent weights so hidden states stay informative."""
  rng = np.random.default_rng(seed)
  u = lambda *s: (rng.uniform(-1, 1, size=s) / np.sqrt(H)).astype(np.float32)
  w = {'depth': depth, 'w1': u(H, H), 'b1': u(H), 'w2': u(D, H), 'b2': u(D), 'h0': u(depth, 1, H),
       'sigma2': (0.05 + 0.1 * rng.random(D)).astype(np.float32), 'transition_bias': p0, 'crp_alpha': alpha}
  for l in range(depth):
    w['weight_ih_l%d' % l] = u(3 * H, D if l == 0 else H)
    w['weight_hh_l%d' % l] = u(3 * H, H)
    w['bias_ih_l%d' % l] = u(3 * H)
    w['bias_hh_l%d' % l] = u(3 * H)
  return w


_MODELS = {}


def model(native, key):
  """(weights, NativeModel, replay Model, kernel mean0) for a fixture name or a random_weights key tuple."""
  if key not in _MODELS:
    if isinstance(key, str):
      w = load_weights(key)
    elif key[0] == 'tiny_sigma2':
      w = dict(load_weights(key[1]))
      w['sigma2'] = (np.asarray(w['sigma2'], np.float32) * np.float32(1e-4)).astype(np.float32)
    else:
      w = random_weights(*key)
    nm = native.NativeModel(w)
    _MODELS[key] = (w, nm, R.Model(w), nm.constants()[0])
  return _MODELS[key]


def synth(seed, n, dim=256, spk=3, noise=0.059):
  from uisrnn_b200.synth import synth_utt
  return synth_utt(seed, n_frames=n, dim=dim, n_spk=spk, noise=noise)[0]


def clustered(rng, n, D, spk=3, run=7, scale=0.3, noise=0.05):
  centres = rng.standard_normal((spk, D))
  return centres[(np.arange(n) // run) % spk] * scale + noise * rng.standard_normal((n, D))


def traced(native, key, xs, kw, expect, trace=None, visit=None, monkeypatch=None, env=None):
  """Decodes xs once per traced utterance (default: all), checks each trace against the replay and every call's
  stats against `expect`.  Returns the replays of the traced utterances."""
  w, nm, rm, mean0 = model(native, key)
  for k, v in (env or {}).items():
    monkeypatch.setenv(k, v)
  mx = kw.get('max_speakers', 0)
  mn = kw.get('min_speakers', 0)
  worst = {}
  out = []
  for u in (range(len(xs)) if trace is None else trace):
    labels, dbg = nm.predict(xs, trace_utt=u, **kw)
    st = nm.stats()
    got = {k: st[k] for k in expect}
    assert got == expect, 'utterance %d ran %s, expected %s' % (u, got, expect)
    rp = R.Replay(rm, xs[u], kw.get('beam_size', 10), kw.get('look_ahead', 1), kw.get('test_iteration', 2),
                  dbg['win'], dbg['score'], dbg['off'], mx if np.ndim(mx) == 0 else mx[u],
                  mn if np.ndim(mn) == 0 else mn[u], mean0=mean0)
    final = dict(best_mean=dbg['best_mean'], best_hidden=dbg['best_hidden'], best_blocks=dbg['best_blocks'],
                 final_k=dbg['final_k'][u], final_scores=dbg['final_scores'][u])
    R.check(rp, INC_RTOL, labels=labels[u].tolist(), final=final if len(xs[u]) else None, state_tol=STATE_TOL,
            worst=worst, visit=visit)
    out.append(rp)
  for k, v in worst.items():
    WORST[k] = max(WORST.get(k, 0.0), v)
  print(' replay worst: ' + ', '.join('%s %.2e' % kv for kv in sorted(worst.items())), end='')
  return out


TOY = 'model_toy100.npz'


def toy_batch(n_utt, seed, n=(60, 90)):
  rng = np.random.default_rng(seed)
  return [synth(seed + i, int(rng.integers(n[0], n[1] + 1))) for i in range(n_utt)]


# ---- the (512, 256) toy model: both engines, lanes, beams

def test_ffma_one_and_two_lanes(native):
  xs = toy_batch(2, 100)
  traced(native, TOY, xs[:1], dict(engine=1, lanes=1, cluster=-1, n_ctas=1),
         dict(engine=1, lanes=1, tc_columns=0, cluster=1, ctas=1))
  traced(native, TOY, xs, dict(engine=1, lanes=2, cluster=-1, n_ctas=1),
         dict(engine=1, lanes=2, tc_columns=0, cluster=1, ctas=1))


@pytest.mark.parametrize('lanes', [6, 3])
def test_tensor_cores_several_lanes(native, lanes):
  """48-column passes shared by 6 lanes per CTA, the most one pass serves, and by 3."""
  xs = toy_batch(lanes, 248)
  traced(native, TOY, xs, dict(engine=2, lanes=lanes, n_ctas=1),
         dict(engine=2, lanes=lanes, tc_columns=48, cluster=1, ctas=1))


def test_tensor_cores_beam_64_two_passes(native):
  """A lane's columns (up to 65) span two 48-column passes."""
  xs = toy_batch(2, 300, n=(30, 40))
  traced(native, TOY, xs, dict(engine=2, lanes=1, n_ctas=2, beam_size=64),
         dict(engine=2, lanes=1, tc_columns=48, cluster=1, ctas=2))


def test_beam_1_tensor_cores_and_beam_128_ffma(native):
  xs = toy_batch(2, 400, n=(40, 50))
  traced(native, TOY, xs, dict(engine=2, lanes=2, n_ctas=1, beam_size=1),
         dict(engine=2, lanes=2, tc_columns=48, cluster=1, ctas=1))
  # (beam 128 shrinks the default kcap to what shared memory holds; max_speakers 4 keeps K below any of them)
  traced(native, TOY, xs[:1], dict(engine=1, lanes=1, cluster=-1, n_ctas=1, beam_size=128, max_speakers=4),
         dict(engine=1, lanes=1, tc_columns=0, cluster=1, ctas=1))


@pytest.mark.parametrize('engine,kcap,lanes', [(1, 24, 2), (2, 16, 3)])
def test_untrained_256x128_near_kcap(native, engine, kcap, lanes):
  """crp_alpha 100 makes an untrained model open a cluster at most frames; max_speakers = kcap lets K reach kcap
  without an overflow."""
  rng = np.random.default_rng(500 + engine)
  xs = [rng.standard_normal((n, 128)) * 0.3 for n in (40, 33, 27)][:lanes]
  key = (256, 128, 1, 256 + 128, 0.5, 100.0)
  traced(native, key, xs,
         dict(engine=engine, lanes=lanes, n_ctas=1, cluster=-1 if engine == 1 else 0, kcap=kcap, max_speakers=kcap),
         dict(engine=engine, lanes=lanes, tc_columns=48 if engine == 2 else 0, cluster=1, ctas=1))
  assert model(native, key)[1].stats()['max_k'] >= kcap - 2


# ---- latency modes

@pytest.mark.parametrize('cluster', [2, 4, 8, 32])
def test_cluster_and_stationary_modes_long(native, cluster):
  x = synth(600 + cluster, 600)
  traced(native, TOY, [x], dict(engine=1, cluster=cluster), dict(engine=1, lanes=1, tc_columns=0, cluster=cluster,
                                                                  ctas=cluster))


# ---- depth

@pytest.mark.parametrize('H,D,depth', [(128, 64, 2), (128, 64, 3), (128, 64, 4), (512, 256, 2), (1024, 512, 1),
                                       (1024, 512, 2)])
def test_depth_and_large_models(native, H, D, depth):
  rng = np.random.default_rng(H + D + depth)
  n = 16 if H == 1024 else 40
  xs = [clustered(rng, n, D), clustered(rng, n // 2 + 1, D)]
  traced(native, (H, D, depth, 7 * H + depth), xs, dict(engine=1, lanes=1, cluster=-1, n_ctas=2, beam_size=5, kcap=64),
         dict(engine=1, lanes=1, tc_columns=0, cluster=1, ctas=2))


# ---- zero-padded shapes

@pytest.mark.parametrize('H,D,depth,engine', [(100, 40, 1, 1), (8, 2, 2, 1), (300, 200, 1, 2), (129, 65, 1, 1),
                                              (600, 300, 1, 1)])
def test_padded_shapes(native, H, D, depth, engine):
  """Replayed at the caller's shape; (300, 200) runs zero-padded on the tensor-core engine at (512, 256)."""
  rng = np.random.default_rng(1000 * H + D)
  xs = [clustered(rng, 31, D), clustered(rng, 18, D)]
  traced(native, (H, D, depth, 1000 * H + D), xs, dict(engine=engine, lanes=1, n_ctas=2, beam_size=5, kcap=64,
                                                        cluster=-1 if engine == 1 else 0),
         dict(engine=engine, lanes=1, tc_columns=48 if engine == 2 else 0, cluster=1, ctas=2))


# ---- look-ahead tree kernel

@pytest.mark.parametrize('spill', ['0', 'force'])
@pytest.mark.parametrize('la', [2, 3])
def test_look_ahead_tree_kernel(native, monkeypatch, la, spill):
  """Shared-memory tree and the spilled tree; 31 frames leave a tail chunk at either look_ahead."""
  from uisrnn_b200.synth import synth_utt
  xs = [synth_utt(700 + i, n_frames=n, dim=64, n_spk=3, noise=0.08)[0] for i, n in enumerate((31, 20))]
  kw = dict(look_ahead=la, beam_size=6, test_iteration=1, n_ctas=2)
  # one tree kernel per call (cast, input projection, tree kernel): without the switch the shared-memory kernel and the
  # spill kernel would both be launched
  traced(native, 'model_small.npz', xs, kw, dict(engine=1, lanes=1, cluster=1, ctas=2, kernel_launches=3),
         monkeypatch=monkeypatch, env={'UISRNN_B200_TREE_SPILL': spill})
  # and only the spill kernel holds its device-memory arenas
  nm = model(native, 'model_small.npz')[1]
  held = workspace_bytes(nm, xs, kw)
  monkeypatch.setenv('UISRNN_B200_TREE_SPILL', '0' if spill == 'force' else 'force')
  assert (held > workspace_bytes(nm, xs, kw)) == (spill == 'force')


def workspace_bytes(nm, xs, kw):
  import ctypes
  off = np.concatenate([[0], np.cumsum([len(x) for x in xs])]).astype(np.int64)
  opts = nm._opts(kw['beam_size'], kw['look_ahead'], kw['test_iteration'], 0, kw['n_ctas'])
  return int(nm._lib.uis_predict_workspace_bytes(nm._h, off.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), len(xs),
                                                 ctypes.byref(opts)))


def test_look_ahead_2_beam_30_toy(native):
  traced(native, TOY, [synth(800, 24)], dict(look_ahead=2, beam_size=30, test_iteration=2),
         dict(engine=1, lanes=1, cluster=1, ctas=1))


# ---- speaker bounds

@pytest.mark.parametrize('engine,mx,mn', [(1, 2, 0), (2, 3, 3), (1, 0, 9)])
def test_speaker_bounds(native, engine, mx, mn):
  """max_speakers 2; max 3 with min 3; a min_speakers no final hypothesis meets (labels from rank 0)."""
  xs = [synth(900 + i, 70, spk=5) for i in range(2)]
  reps = traced(native, TOY, xs, dict(engine=engine, lanes=2, n_ctas=1, max_speakers=mx, min_speakers=mn,
                                      cluster=-1 if engine == 1 else 0),
                dict(engine=engine, lanes=2, tc_columns=48 if engine == 2 else 0, cluster=1, ctas=1))
  if mn == 9:
    assert all(rp.chosen() == 0 and rp.hyps[0].K < mn for rp in reps)
  if mx:
    assert all(h.K <= mx for rp in reps for h in rp.hyps)


# ---- long decodes: 4200 steps, beyond the 4094 the default log tables hold

@pytest.mark.parametrize('engine', [2, 1])
def test_long_decode_4200_steps(native, engine):
  x = synth(1000 + engine, 2100)
  traced(native, TOY, [x], dict(engine=engine, lanes=1, n_ctas=1, cluster=-1 if engine == 1 else 0),
         dict(engine=engine, lanes=1, tc_columns=48 if engine == 2 else 0, cluster=1, ctas=1))


def test_alternating_speakers_past_4096_turns(native):
  """Two speakers alternating every frame: the best hypothesis changes cluster at every step, so its ddCRP
  denominator log(turns + alpha) reads the regrown log table past its default 4096 entries."""
  rng = np.random.default_rng(1050)
  c = rng.standard_normal((2, 256))
  c *= 2.0 / np.linalg.norm(c, axis=1, keepdims=True)
  x = c[np.arange(2100) % 2] + 0.01 * rng.standard_normal((2100, 256))
  rp, = traced(native, TOY, [x], dict(engine=2, lanes=1, n_ctas=1), dict(engine=2, lanes=1, tc_columns=48, cluster=1,
                                                                         ctas=1))
  assert sum(rp.hyps[0].blocks) > 4096


# ---- host staging chunks

def test_host_staging_chunks(native, monkeypatch):
  """256-row staging chunks: chunk boundaries fall inside both traced utterances."""
  xs = [synth(1100, 300), synth(1101, 500)]
  traced(native, TOY, xs, dict(engine=2, lanes=2, n_ctas=1), dict(engine=2, lanes=2, tc_columns=48, cluster=1, ctas=1),
         monkeypatch=monkeypatch, env={'UISRNN_B200_CHUNK_MB': '0'})
  assert model(native, TOY)[1].stats()['chunks'] >= 3


def test_staging_chunk_first_row_is_rounded_to_nearest(native, monkeypatch):
  """The first row of the second 256-row staging chunk (frame 56 of the second utterance) equals the kernel's mean0
  except that x[0] lies 0.4 of an fp32 spacing below mean0[0] in magnitude: rounded to nearest it is mean0[0], so every
  new-cluster candidate at that frame is +inf; any other rounding (toward zero, say) would make a new cluster the clear
  winner there."""
  _, _, _, mean0 = model(native, TOY)
  m = np.float32(mean0[0])
  xs = [synth(1150, 200), synth(1151, 300)]
  xs[1][56] = mean0
  xs[1][56, 0] = float(m) + 0.4 * (float(np.nextafter(m, np.float32(0))) - float(m))
  assert np.float32(xs[1][56, 0]) == m
  reps = traced(native, TOY, xs, dict(engine=2, lanes=2, n_ctas=1),
                dict(engine=2, lanes=2, tc_columns=48, cluster=1, ctas=1), trace=[1], monkeypatch=monkeypatch,
                env={'UISRNN_B200_CHUNK_MB': '0'})
  assert model(native, TOY)[1].stats()['chunks'] == 2 and len(reps) == 1


# ---- edge inputs

@pytest.mark.parametrize('engine', [1, 2])
def test_edge_inputs(native, engine):
  """0-, 1- and 2-frame utterances, all-zero frames and a frame x1e3, beside a frame whose x[0] equals the kernel's
  mean0[0] in fp32: there every new-cluster candidate is +inf, and fewer than beam_size candidates are finite."""
  _, _, _, mean0 = model(native, TOY)
  a = synth(1200, 30)
  a[5:8] = 0.0
  big = synth(1204, 30)
  big[12] *= 1e3
  b = synth(1201, 20)
  b[2, 0] = float(mean0[0])
  xs = [np.zeros((0, 256)), synth(1202, 1), synth(1203, 2), a, big, b]
  seen = []

  def at_frame_2(s, st):
    if s == 2 and st.inc.shape[0] == 2:
      new = [st.inc[p, h.K] for p, h in enumerate(st_prev[0])]
      seen.append((all(np.isinf(new)), len(st.rows)))
    st_prev[0] = st.hyps
  st_prev = [None]
  kw = dict(engine=engine, lanes=2, n_ctas=1, cluster=-1 if engine == 1 else 0)
  expect = dict(engine=engine, lanes=2, tc_columns=48 if engine == 2 else 0, cluster=1, ctas=1)
  traced(native, TOY, xs, kw, expect, trace=[1, 2, 3, 4])
  traced(native, TOY, xs, kw, expect, trace=[5], visit=at_frame_2)
  assert seen == [(True, 3)]  # hypotheses (0, 0) and (0, 1): 2 + 3 candidates, the 2 new-cluster ones +inf
  labels = model(native, TOY)[1].predict(xs, **kw)
  assert len(labels[0]) == 0


def test_tiny_sigma2(native):
  traced(native, ('tiny_sigma2', TOY), toy_batch(2, 1300, n=(30, 40)), dict(engine=2, lanes=2, n_ctas=1),
         dict(engine=2, lanes=2, tc_columns=48, cluster=1, ctas=1))


def test_report_worst():
  """Runs last in this file: the worst error per class over every case above (shown with -s)."""
  print('\nkernel vs float64 replay, worst: ' + ', '.join('%s %.2e' % kv for kv in sorted(WORST.items())))
  if WORST:
    assert WORST['inc'] <= INC_RTOL and WORST['mean'] <= STATE_TOL and WORST['hidden'] <= STATE_TOL
