"""The float64 step replay (tests/beam_replay.py) pinned without a GPU: every traced golden the unmodified reference
produced, and oracle records on fresh inputs, pass its step, selection, state and label checks at the bounds below;
and traces perturbed in the ways a kernel could go wrong fail them.  The path rescorer (beam_replay.path_score) is
pinned the same way: every final rank of every traced golden, rescored from its labels alone, lies within the allowance
of the reference's fp32 score (worst: 0.17 of it), and a relabelled frame or a score moved past the allowance fails.

The reference's own fp32 search is what the replay is measured against here.  Its worst deviation over this file
(printed by test_report_worst with `pytest -s`) is beside each bound; the bounds are about 10x that."""
import numpy as np
import pytest

import beam_replay as R
from helpers import GOLDEN, depth2_cases, load_weights, oracle_model, rel_err, small_cases, toy_utterances, uis_oracle
import speaker_bounds_oracle as SB
from test_speaker_bounds_cpu import CASES as BOUND_CASES

REF_INC_RTOL = 5e-7     # increment beyond la ulp of the score, relative to |increment|: 5.3e-8
REF_STATE_TOL = 5e-6    # best_mean / best_hidden rows, relative to the row's largest value: 4.4e-7
WORST = {}


def golden_cases():
  out = []
  xs, _ = toy_utterances()
  g = np.load(GOLDEN + '/toy_trace.npz')
  for i in (0, 1):
    k = lambda s: g['u%d_%s' % (i, s)]
    out.append(dict(name='toy_u%d' % i, model='model_toy100.npz', x=xs[i], beam_size=10, look_ahead=1,
                    test_iteration=2, win=k('win'), score=k('score'), off=k('off'), labels=k('labels'),
                    final_mean=k('final_mean'), final_hidden=k('final_hidden'), final_blocks=k('final_blocks')))
  for cases, model in ((small_cases(), 'model_small.npz'), (depth2_cases(), 'model_small_d2.npz')):
    for c in cases:
      out.append(dict(c, model=model))
  for c in BOUND_CASES:
    out.append(dict(c, name='bounds_' + c['name']))
  return out


GOLDEN_CASES = golden_cases()


def run(case, worst=WORST, labels=True):
  rp = R.Replay(load_weights(case['model']), case['x'], case['beam_size'], case['look_ahead'], case['test_iteration'],
                case['win'], case['score'], case['off'], case.get('max_speakers', 0), case.get('min_speakers', 0))
  final = None
  if 'final_mean' in case:
    off = case['off']
    final = dict(best_mean=case['final_mean'], best_hidden=case['final_hidden'], best_blocks=case['final_blocks'],
                 final_k=len(case['final_blocks']), final_scores=case['score'][off[-2]:off[-1]])
  return R.check(rp, REF_INC_RTOL, labels=case['labels'].tolist() if labels else None, final=final,
                 state_tol=REF_STATE_TOL, worst=worst)


@pytest.mark.parametrize('case', GOLDEN_CASES, ids=[c['name'] for c in GOLDEN_CASES])
def test_reference_goldens_pass_the_replay(case):
  """Toy trace, small_cases (look_ahead 1-3, beams 1-30), depth2_cases and speaker_bounds_cases: step, selection and
  (where recorded) state checks; the back-track of the trace gives the golden labels."""
  run(case)


def fresh_cases():
  from uisrnn_b200.synth import synth_utt
  out = []
  for i, (n, spk, b, la, ti, mx, mn) in enumerate([(90, 3, 10, 1, 2, 0, 0), (41, 4, 6, 2, 1, 0, 0),
                                                    (32, 3, 4, 3, 2, 0, 0), (60, 5, 8, 1, 2, 2, 0),
                                                    (25, 4, 5, 2, 2, 3, 3)]):
    x = synth_utt(8100 + i, n_frames=n, dim=64, n_spk=spk, noise=0.08)[0]
    rec = {}
    labels = SB.predict_single(oracle_model('model_small.npz'), x, b, la, ti, max_speakers=mx, min_speakers=mn,
                               record=rec)
    out.append(dict(name='fresh%d_b%d_la%d' % (i, b, la), model='model_small.npz', x=x, beam_size=b, look_ahead=la,
                    test_iteration=ti, max_speakers=mx, min_speakers=mn, labels=np.array(labels), **rec))
  return out


def test_fresh_oracle_records_pass_the_replay():
  """Oracle records on inputs no golden holds, with and without bounds, a tail chunk (32 frames x 2 at look_ahead 3)."""
  for case in fresh_cases():
    run(case)


def toy_case():
  return dict(GOLDEN_CASES[0])


def test_late_score_moved_by_1e6_fails():
  """1e-6 of the score is within the 1e-5 relative score check of compare_trace, but is many increments' tolerance."""
  case = toy_case()
  off = case['off']
  r = int(off[len(off) - 10])
  score = case['score'].copy()
  score[r] = float(np.float32(score[r] * (1 + 1e-6)))
  assert rel_err(score, case['score']) < 1e-5
  with pytest.raises(AssertionError, match='increment'):
    run(dict(case, score=score), worst={})


def test_winners_swapped_across_a_gap_fail():
  case = toy_case()
  off, win = case['off'], case['win'].copy()
  s = len(off) // 2
  lo = int(off[s])
  assert case['score'][lo + 1] - case['score'][lo] > 1.0  # a real gap between ranks 0 and 1 at this step
  win[[lo, lo + 1]] = win[[lo + 1, lo]]
  with pytest.raises(AssertionError):
    run(dict(case, win=win), worst={}, labels=False)


def test_dropped_finite_winner_fails():
  case = toy_case()
  off = case['off'].copy()
  off[-1] -= 1
  n = int(off[-1])
  case = dict(case, win=case['win'][:n], score=case['score'][:n], off=off)
  del case['final_mean']
  with pytest.raises(AssertionError, match='winners'):
    run(case, worst={}, labels=False)


def test_cluster_beyond_max_speakers_fails():
  case = next(c for c in GOLDEN_CASES if c['name'] == 'bounds_s_b10_la1_t2')
  mx, win, off = case['max_speakers'], case['win'].copy(), case['off']
  assert mx and case['look_ahead'] == 1
  k_prev = [0]
  for s in range(len(off) - 1):
    k_now = []
    for r in range(int(off[s]), int(off[s + 1])):
      b, c = int(win[r, 0]), int(win[r, 1])
      if k_prev[b] == mx and c < mx:  # open one cluster too many instead
        win[r, 1] = mx
        with pytest.raises(AssertionError, match=r'\+inf'):
          run(dict(case, win=win), worst={}, labels=False)
        return
      k_now.append(k_prev[b] + (c == k_prev[b]))
    k_prev = k_now
  pytest.fail('no hypothesis at the bound')


def test_replay_keeps_first_column_rule():
  """x[0] equal to mean0[0] in fp32: with the kernel's mean0 given, every new-cluster candidate is +inf; without it
  they are undecided, never silently finite."""
  w = load_weights('model_small.npz')
  om = oracle_model('model_small.npz')
  from uisrnn_b200.synth import synth_utt
  x = synth_utt(8200, n_frames=12, dim=64, n_spk=3, noise=0.08)[0]
  x[2, 0] = float(om.mean0[0])
  rec = {}
  labels = uis_oracle.predict_single(om, x, beam_size=10, look_ahead=1, test_iteration=1, record=rec)
  assert rec['nfinite'][2] < rec['nfinite'][2 - 1] + 3  # the oracle drops the new-cluster candidates at frame 2
  for mean0 in (om.mean0, None):
    rp = R.Replay(w, x, 10, 1, 1, rec['win'], rec['score'], rec['off'], mean0=mean0)
    for st in rp.steps():
      if st.t == 2:
        new = [st.inc[(b,) + (h.K,)] for b, h in enumerate(st_hyps)]
        amb = [st.ambiguous[(b,) + (h.K,)] for b, h in enumerate(st_hyps)]
        assert all(np.isinf(new)) if mean0 is not None else all(amb)
        assert int((np.isfinite(st.inc) & ~st.ambiguous).sum()) == rec['nfinite'][2] or mean0 is None
      st_hyps = st.hyps
    assert R.check(R.Replay(w, x, 10, 1, 1, rec['win'], rec['score'], rec['off'], mean0=mean0), REF_INC_RTOL) == labels


def final_paths(case):
  """Every final rank of a traced golden as (tiled x, labels [R, N * test_iteration], the reference's fp32 final
  scores [R]): the back-track of the trace from each rank, over the whole tiled decode."""
  off, T = case['off'], case['test_iteration']
  tn = len(case['x']) * T
  finals = int(off[-1] - off[-2])
  labels = np.array([R.backtrack(case['win'], off, tn, r) for r in range(finals)], np.int64).reshape(finals, tn)
  return np.tile(case['x'], (T, 1)), labels, case['score'][int(off[-2]):int(off[-1])].astype(np.float64)


def rescore(case, worst=None):
  x, labels, ref = final_paths(case)
  res = R.path_score(load_weights(case['model']), [x], [labels])
  used = res.share(ref, REF_INC_RTOL)
  if worst is not None:
    worst['path'] = max(worst.get('path', 0.0), float(used.max()))
  return labels, ref, res, used


@pytest.mark.parametrize('case', GOLDEN_CASES, ids=[c['name'] for c in GOLDEN_CASES])
def test_rescored_final_ranks_match_reference(case):
  """Every final rank of every traced golden (toy trace, small_cases, depth2_cases, speaker_bounds_cases: look_ahead
  1-3, test_iteration 1-3, with and without bounds) rescored from its labels alone lies within the allowance of the
  reference's own fp32 score; the recorded final traces and golden labels are the last tiled copy of those paths."""
  labels, ref, res, used = rescore(case, WORST)
  r = int(np.argmax(used))
  assert used[r] <= 1, 'rank %d: score %.9g, float64 %.12g, allowed %.3g' % (r, ref[r], res.score[r],
                                                                             res.allowance(REF_INC_RTOL)[r])
  last = labels[:, labels.shape[1] - len(case['x']):]
  if 'final_traces' in case:
    assert np.array_equal(last, case['final_traces'][:len(labels)])
  assert last[int(case.get('chosen', 0))].tolist() == case['labels'].tolist()


def test_relabelled_frame_fails_the_rescore():
  """Rank 0 of a 60-frame decode with every single frame moved to another cluster it could have joined: each of these
  paths scores outside the allowance of the reference's rank-0 score."""
  case = next(c for c in GOLDEN_CASES if c['name'] == 'bounds_s_min_pick')
  x, labels, ref = final_paths(case)
  path = labels[0]
  moved = []
  for t in range(1, len(path)):
    opened = int(path[:t].max()) + 1
    if path[t] < opened and opened > 1:  # (not the frame that opens its cluster: the clusters still open in order)
      q = path.copy()
      q[t] = (path[t] + 1) % opened
      moved.append(q)
  assert len(moved) > 25
  res = R.path_score(load_weights(case['model']), [x], [np.array(moved)])
  assert np.all(np.abs(res.score - ref[0]) > res.allowance(REF_INC_RTOL))


def test_final_score_moved_past_the_allowance_fails():
  """The final score of the longest traced decode (180 sub-steps) moved by 4 fp32 ulps beyond its allowance: still
  inside a 1e-5 relative score check, outside the rescore.  (The allowance itself holds one ulp of the running score
  per sub-step, about half the decode's length in ulps of the final score.)"""
  case = next(c for c in GOLDEN_CASES if c['name'] == 'b10')
  x, labels, ref = final_paths(case)
  res = R.path_score(load_weights(case['model']), [x], [labels[:1]])
  s = np.float32(ref[0])
  assert res.share(ref[:1], REF_INC_RTOL)[0] <= 1
  moved = np.float32(res.score[0] + np.sign(s - res.score[0]) * res.allowance(REF_INC_RTOL)[0])
  for _ in range(4):
    moved = np.nextafter(moved, np.float32(np.inf) if moved > res.score[0] else np.float32(-np.inf))
  assert rel_err([moved], [s]) < 1e-5
  assert res.share([float(moved)], REF_INC_RTOL)[0] > 1
  assert res.allowance(REF_INC_RTOL)[0] < 200 * float(R.ulp32(s))


def test_rescore_batches_and_shares_states():
  """Paths rescored together, with duplicates, absent ranks and an empty utterance, score as they do alone."""
  a = next(c for c in GOLDEN_CASES if c['name'] == 'b10')
  b = next(c for c in GOLDEN_CASES if c['name'] == 'la3')
  xa, la, _ = final_paths(a)
  xb, lb, _ = final_paths(b)
  w = load_weights('model_small.npz')
  alone = [R.path_score(w, [xa], [la]), R.path_score(w, [xb], [lb])]
  lb_absent = np.concatenate([lb, np.full((2, lb.shape[1]), -1)])
  together = R.path_score(w, [xb, np.zeros((0, 64)), xa], [lb_absent, np.zeros((1, 0), np.int64), np.concatenate([la, la])],
                          max_slots=20)
  nb = len(lb)
  for got, want in ((together.score[:nb], alone[1].score), (together.score[nb + 3:nb + 3 + len(la)], alone[0].score),
                    (together.score[nb + 3 + len(la):], alone[0].score), (together.ulps[:nb], alone[1].ulps)):
    assert np.array_equal(got, want)
  assert np.isnan(together.score[nb:nb + 2]).all() and together.score[nb + 2] == 0


def test_report_worst():
  """The replay's measured deviation from the reference's fp32 search (run with -s to see it)."""
  worst = {}
  for case in GOLDEN_CASES:
    run(case, worst=worst)
    rescore(case, worst)
  print('\nreference vs float64 replay, worst: ' + ', '.join('%s %.2e' % kv for kv in sorted(worst.items())))
  assert worst['inc'] <= REF_INC_RTOL and worst['mean'] <= REF_STATE_TOL and worst['hidden'] <= REF_STATE_TOL
  assert worst['path'] <= 1
