"""Full-occupancy predict() calls and the device entry point pinned to float64, per utterance and per returned rank.

test_gpu_step_replay.py replays traced utterances of calls on one or two CTAs.  Here the calls are shaped like the ones
users make (bench.py times 792 x 500 frames): the automatic plan on every SM with more utterances than lanes, so that
lanes are refilled from the longest-first queue, beside every other CTA sharing L2 and the queue.  The batch is ragged
(0-600 frames, mostly distinct lengths, 0-, 1- and 2-frame utterances included).

a. Traced utterances inside such calls, checked per beam step by beam_replay.check: the shortest utterances (the
   queue hands them out last, so each goes to a lane that has already finished one) and two from the middle of the
   queue; on the tensor-core engine, the FFMA engine (2 lanes), with per-utterance speaker bounds, and through the
   look-ahead tree kernel (beam 30, look_ahead 2) in shared memory and in the spill kernel's own queue.  Every traced
   utterance is asserted to sit past the first lanes x CTAs positions of the queue.  (A traced call never decodes in
   groups: decode-in-groups is covered by (b) and (c).)
b. Every utterance and every rank (n_best = beam_size) bit-identical across call composition, per engine: the list
   permuted, 61 and 7 CTAs, 4 and 1 lanes, 256-row staging chunks, pageable inputs staged by the driver instead of the
   pinned ring, decode in groups, and predict_device_nbest on a non-default stream (what bench.py times); plane 0
   equals the call without n_best.  A column's arithmetic does not depend on the lane, pass position or CTA it lands
   in, nor the input projection on a row's position in its tile.  Engines and the
   cluster / stationary-weights modes are not compared with each other: they split k differently.  That includes a
   group of a decode-in-groups call: each group is planned on its own, and a group of no more utterances than SMs
   runs a latency-mode kernel under the automatic plan (a split of the rows in thirds left the last 3 utterances to
   the 4-CTA cluster kernel: 1-ulp score differences and one near-tied rank swapped), so the groups here hold more.
c. Every returned hypothesis of the test_iteration-1 calls rescored from its labels (beam_replay.path_score): its
   fp32 score within the allowance of an fp32 accumulation, scores non-decreasing by rank, speakers = the distinct
   labels of the rank, count = min(n_best, #distinct paths), absent ranks +inf / -1 / 0.

Every call asserts which kernel ran (stats: engine, lanes, tensor-core columns, cluster, CTAs, utterances).  The
untraced utterances of test_iteration-2 calls are bit-compared only: their returned labels are the last tiled copy,
which does not determine the path."""
import numpy as np
import pytest

import beam_replay as R
from test_gpu_step_replay import model, synth

pytestmark = pytest.mark.gpu

INC_RTOL, STATE_TOL = R.INC_RTOL, R.STATE_TOL
TOY = 'model_toy100.npz'
U_FULL = 1100
# worst error per class over this file: replay ('inc', 'mean', 'hidden') and the share of its allowance a returned
# score uses ('path')
WORST = {}


@pytest.fixture(scope='module')
def native():
  from uisrnn_b200 import native as nat
  nat.load_library()
  return nat


@pytest.fixture(scope='module')
def sms():
  import torch
  return torch.cuda.get_device_properties(0).multi_processor_count


def ragged(seed, U, longest):
  """U utterances of the toy model's dimension: 0, 1 and 2 frames, every length 3..longest once, then random ones."""
  rng = np.random.default_rng(seed)
  n = np.concatenate([[0, 1, 2], rng.permutation(np.arange(3, longest + 1)), rng.integers(3, longest + 1, U)])[:U]
  n = rng.permutation(n)
  return [synth(100 * seed + i, int(k)) if k else np.zeros((0, 256)) for i, k in enumerate(n)]


@pytest.fixture(scope='module')
def batch():
  return ragged(71, U_FULL, 600)


def queue_position(xs):
  """Position of every utterance in the kernels' queue (longest first, stable)."""
  n = [len(x) for x in xs]
  pos = np.empty(len(xs), np.int64)
  pos[sorted(range(len(xs)), key=lambda u: -n[u])] = np.arange(len(xs))
  return pos


def pick_traced(xs, refilled_from):
  """The three shortest non-empty utterances (handed out last) and two from the middle of the refill part."""
  pos = queue_position(xs)
  by_pos = np.argsort(pos)
  short = [int(u) for u in by_pos[::-1] if len(xs[u])][:3]
  mid = [int(by_pos[(len(xs) + refilled_from) // 2]), int(by_pos[refilled_from + (len(xs) - refilled_from) // 4])]
  return short + mid


def check_stats(nm, expect, what=''):
  st = nm.stats()
  got = {k: st[k] for k in expect}
  assert got == expect, '%s ran %s, expected %s' % (what, got, expect)
  return st


def traced_calls(native, xs, kw, expect, trace, max_speakers=None, min_speakers=None, T=2):
  """One call per traced utterance, each checked per step against the float64 replay and the plain call's labels."""
  w, nm, rm, mean0 = model(native, TOY)
  bounds = dict(max_speakers=max_speakers, min_speakers=min_speakers)
  plain = nm.predict(xs, test_iteration=T, **bounds, **kw)
  check_stats(nm, expect, 'the plain call')
  pos = queue_position(xs)
  worst = {}
  for u in trace:
    assert pos[u] >= expect['lanes'] * expect['ctas'], 'utterance %d is not decoded by a refilled lane' % u
    labels, dbg = nm.predict(xs, trace_utt=u, test_iteration=T, **bounds, **kw)
    check_stats(nm, expect, 'utterance %d' % u)
    assert all(np.array_equal(a, b) for a, b in zip(labels, plain)), 'a traced call returns other labels'
    rp = R.Replay(rm, xs[u], kw.get('beam_size', 10), kw.get('look_ahead', 1), T, dbg['win'], dbg['score'],
                  dbg['off'], 0 if max_speakers is None else max_speakers[u],
                  0 if min_speakers is None else min_speakers[u], mean0=mean0)
    final = dict(best_mean=dbg['best_mean'], best_hidden=dbg['best_hidden'], best_blocks=dbg['best_blocks'],
                 final_k=dbg['final_k'][u], final_scores=dbg['final_scores'][u])
    R.check(rp, INC_RTOL, labels=labels[u].tolist(), final=final, state_tol=STATE_TOL, worst=worst)
  for k, v in worst.items():
    WORST[k] = max(WORST.get(k, 0.0), v)
  print(' replay worst: ' + ', '.join('%s %.2e' % kv for kv in sorted(worst.items())), end='')
  return plain


def tc_plan(sms, U=U_FULL, lanes=6):
  return dict(engine=2, lanes=lanes, tc_columns=48, cluster=1, ctas=sms, utterances=U)


def ffma_plan(sms, lanes, U=U_FULL, ctas=None):
  return dict(engine=1, lanes=lanes, tc_columns=0, cluster=1, ctas=ctas or sms, utterances=U)


# ---- a. traced utterances inside full-occupancy calls

def test_traced_tensor_cores_automatic_plan(native, batch, sms):
  assert U_FULL > 6 * sms
  traced_calls(native, batch, {}, tc_plan(sms), pick_traced(batch, 6 * sms))


def test_traced_ffma_two_lanes(native, batch, sms):
  traced_calls(native, batch, dict(engine=1, lanes=2, cluster=-1), ffma_plan(sms, 2), pick_traced(batch, 2 * sms))


def test_traced_per_utterance_speaker_bounds(native, batch, sms):
  """Mixed bounds, so that a refilled lane usually changes them: max in {0, 1, 2, 3, 5}, min up to max."""
  rng = np.random.default_rng(72)
  mx = rng.choice([0, 1, 2, 3, 5], U_FULL).astype(np.int32)
  mn = np.where(mx > 0, rng.integers(0, mx + 1), rng.integers(0, 4, U_FULL)).astype(np.int32)
  trace = pick_traced(batch, 6 * sms)
  assert len({(int(mx[u]), int(mn[u])) for u in trace}) > 2
  plain = traced_calls(native, batch, {}, tc_plan(sms), trace, max_speakers=mx, min_speakers=mn)
  for u, lab in enumerate(plain):
    assert mx[u] == 0 or len(lab) == 0 or lab.max() < mx[u], u


@pytest.mark.parametrize('spill', ['0', 'force'])
def test_traced_look_ahead_tree_kernel(native, monkeypatch, sms, spill):
  """Config-3 shape (beam 30, look_ahead 2) on every SM: each CTA pulls several utterances, from the shared-memory
  kernel's queue or from the spill kernel's second queue.  Every rank rescored (test_iteration 1)."""
  monkeypatch.setenv('UISRNN_B200_TREE_SPILL', spill)
  xs = ragged(73, 300, 150)
  kw = dict(beam_size=30, look_ahead=2)
  expect = dict(engine=1, lanes=1, cluster=1, ctas=sms, utterances=300)
  traced_calls(native, xs, kw, expect, pick_traced(xs, sms), T=1)
  w, nm, rm, mean0 = model(native, TOY)
  out = nm.predict(xs, test_iteration=1, n_best=30, **kw)
  st = check_stats(nm, expect, 'the n-best call')
  # one tree kernel (a cast and an input projection per staging chunk): without the switch the shared-memory kernel
  # and the spill kernel would both be launched
  assert st['kernel_launches'] == 2 * st['chunks'] + 1
  rescore_all(rm, mean0, xs, out, 30)


# ---- b. and c. bit identity across call composition, every rank rescored

VARIANTS = {'tc': dict(), 'ffma2': dict(engine=1, lanes=2, cluster=-1), 'ffma1': dict(engine=1, lanes=1, cluster=-1)}


def same(a, b, what):
  """Labels of every plane, scores (bits), speakers and count of two n-best results."""
  la, sa, pa, ca = a
  lb, sb, pb, cb = b
  for u in range(len(la)):
    assert np.array_equal(la[u], lb[u]), '%s: utterance %d, labels differ' % (what, u)
  assert np.array_equal(sa.view(np.int32), sb.view(np.int32)), '%s: scores differ (utterance %d)' % (
      what, int(np.argmax(np.any(sa.view(np.int32) != sb.view(np.int32), axis=1))))
  assert np.array_equal(pa, pb) and np.array_equal(ca, cb), '%s: speakers or count differ' % what


def distinct_paths(n):
  """Label paths of n frames (clusters opened in order): the Bell numbers."""
  row = [1]
  for _ in range(n):
    nxt = [row[-1]]
    for v in row:
      nxt.append(nxt[-1] + v)
    row = nxt
  return row[0]


def rescore_all(rm, mean0, xs, out, k):
  """c. for a test_iteration-1 n-best result: every rank against path_score, ranks, speakers, count, absent ranks."""
  labels, scores, speakers, count = out
  for u, x in enumerate(xs):
    c = int(count[u])
    assert c == (min(k, distinct_paths(min(len(x), 8))) if len(x) else 0), 'utterance %d: count %d' % (u, c)
    assert (labels[u][c:] == -1).all() and np.isinf(scores[u][c:]).all() and (speakers[u][c:] == 0).all(), u
    assert np.all(np.diff(scores[u][:c].astype(np.float64)) >= 0), 'utterance %d: ranks out of order' % u
    for j in range(c):
      assert speakers[u][j] == len(set(labels[u][j].tolist())) == labels[u][j].max() + 1, (u, j)
  res = R.path_score(rm, xs, labels, mean0=mean0, device='cuda')
  got = np.concatenate([scores[u][:len(labels[u])] for u in range(len(xs))]).astype(np.float64)
  present = ~np.isnan(res.score) & (np.repeat([len(x) for x in xs], [len(lab) for lab in labels]) > 0)
  used = res.share(got, INC_RTOL)[present]
  WORST['path'] = max(WORST.get('path', 0.0), float(used.max()))
  bad = int(np.argmax(used))
  assert used[bad] <= 1, 'path %d: score %.9g, float64 %.12g, allowed %.3g' % (
      bad, got[present][bad], res.score[present][bad], res.allowance(INC_RTOL)[present][bad])
  print(' rescored %d paths, worst share of the allowance %.2e' % (int(present.sum()), used.max()), end='')


def device_nbest(nm, xs, k, kw):
  """predict_device_nbest on a non-default torch stream, as bench.py calls predict_device."""
  import torch
  off = np.zeros(len(xs) + 1, np.int64)
  np.cumsum([len(x) for x in xs], out=off[1:])
  x = torch.from_numpy(np.concatenate(xs).astype(np.float32)).cuda()
  lab = torch.full((k, int(off[-1])), -7, dtype=torch.int32, device='cuda')
  sc = torch.zeros((len(xs), k), dtype=torch.float32, device='cuda')
  sp = torch.zeros((len(xs), k), dtype=torch.int32, device='cuda')
  cnt = torch.zeros(len(xs), dtype=torch.int32, device='cuda')
  torch.cuda.synchronize()
  side = torch.cuda.Stream()
  nm.predict_device(x.data_ptr(), off, lab.data_ptr(), stream=side.cuda_stream, n_best=k, scores_ptr=sc.data_ptr(),
                    nbest_speakers_ptr=sp.data_ptr(), count_ptr=cnt.data_ptr(), **kw)
  side.synchronize()
  lab = lab.cpu().numpy()
  return [lab[:, off[u]:off[u + 1]] for u in range(len(xs))], sc.cpu().numpy(), sp.cpu().numpy(), cnt.cpu().numpy()


def group_sizes(xs, max_rows):
  """Utterances per group of a call decoded in groups of at most max_rows frames (consecutive whole utterances)."""
  off = np.concatenate([[0], np.cumsum([len(x) for x in xs])])
  sizes, u0 = [], 0
  while u0 < len(xs):
    u1 = u0 + 1
    while u1 < len(xs) and off[u1 + 1] - off[u0] <= max_rows:
      u1 += 1
    sizes.append(u1 - u0)
    u0 = u1
  return sizes


@pytest.mark.parametrize('variant,T', [('tc', 2), ('tc', 1), ('ffma2', 1), ('ffma1', 1)])
def test_call_composition_bit_identical(native, monkeypatch, batch, sms, variant, T):
  w, nm, rm, mean0 = model(native, TOY)
  xs, k = batch, 10
  kw = dict(VARIANTS[variant], test_iteration=T)
  lanes = dict(VARIANTS[variant]).get('lanes', 6)
  plan = tc_plan(sms) if variant == 'tc' else ffma_plan(sms, lanes)
  run = lambda seqs=xs, **over: nm.predict(seqs, n_best=k, **dict(kw, **over))
  ref = run()
  st = check_stats(nm, plan, 'the automatic call')
  assert st['staged'] == 1 and st['groups'] == 1
  if variant == 'tc' and T == 2:
    print(' stats of the automatic call: ' + ', '.join('%s %s' % (q, st[q]) for q in (
        'engine', 'lanes', 'tc_columns', 'cluster', 'ctas', 'utterances', 'beam_steps', 'max_k')), end='')
  plain = nm.predict(xs, **kw)
  assert all(np.array_equal(ref[0][u][0], plain[u]) for u in range(len(xs))), 'plane 0 differs from the plain call'
  # the list permuted
  perm = np.random.default_rng(74).permutation(len(xs))
  got = run([xs[i] for i in perm])
  check_stats(nm, plan, 'the permuted call')
  inv = np.argsort(perm)
  same(ref, ([got[0][i] for i in inv], got[1][inv], got[2][inv], got[3][inv]), 'permuted list')
  # CTAs and lanes
  for ctas in (61, 7):
    same(ref, run(n_ctas=ctas), '%d CTAs' % ctas)
    check_stats(nm, dict(plan, ctas=ctas), '%d CTAs' % ctas)
  if variant == 'tc':
    for g in (4, 1):
      same(ref, run(engine=2, lanes=g), '%d lanes' % g)
      check_stats(nm, tc_plan(sms, lanes=g), '%d lanes' % g)
  # host staging: 256-row chunks, pageable inputs copied by the driver, decode in groups
  monkeypatch.setenv('UISRNN_B200_CHUNK_MB', '0')
  same(ref, run(), '256-row staging chunks')
  assert check_stats(nm, plan)['chunks'] >= sum(len(x) for x in xs) // 256
  monkeypatch.delenv('UISRNN_B200_CHUNK_MB')
  monkeypatch.setenv('UISRNN_B200_HOST_STAGING', '0')
  same(ref, run(), 'driver-staged pageable inputs')
  assert check_stats(nm, plan)['staged'] == 0
  monkeypatch.delenv('UISRNN_B200_HOST_STAGING')
  max_rows = int(sum(len(x) for x in xs) / 2.5) + 1
  groups = group_sizes(xs, max_rows)
  assert len(groups) == 3 and min(groups) > sms
  monkeypatch.setenv('UISRNN_B200_MAX_ROWS', str(max_rows))
  same(ref, run(), 'decode in groups')
  assert nm.stats()['groups'] == 3
  monkeypatch.delenv('UISRNN_B200_MAX_ROWS')
  # the device entry point on a non-default stream
  same(ref, device_nbest(nm, xs, k, kw), 'predict_device_nbest')
  check_stats(nm, plan, 'predict_device_nbest')
  if T == 1:  # c. (the device call's results are bit-identical to these)
    rescore_all(rm, mean0, xs, ref, k)


def test_report_worst():
  """Runs last in this file: the worst error per class over every case above (shown with -s)."""
  print('\nfull occupancy vs float64, worst: ' + ', '.join('%s %.2e' % kv for kv in sorted(WORST.items())))
  if WORST:
    assert WORST.get('inc', 0) <= INC_RTOL and WORST.get('mean', 0) <= STATE_TOL
    assert WORST.get('hidden', 0) <= STATE_TOL and WORST.get('path', 0) <= 1
