#!/usr/bin/env python3
"""Writes tests/golden/speaker_bounds_cases.npz by RUNNING THE REFERENCE'S OWN PREDICT CODE with speaker bounds.

The reference has no speaker bounds.  Its beam search is run unmodified except that the model's `_calculate_score`
(uisrnn.py:455-477) is wrapped: every finite index tuple whose `_update_beam_state(...)` would leave more than
max_speakers entries in `mean_set` gets +inf.  The labels come from the reference's own `predict_single`; the
per-step trace and every final rank (trace, cluster count, score) come from the same control flow as
oracle/make_golden.py's `traced_predict`, driven through the reference's methods, with min_speakers applied at the
end: the first final rank with at least min_speakers clusters, else rank 0.

Cases with max_speakers > 0 are chosen so that the bound binds: the unbounded reference labels open more clusters
than max_speakers (asserted).  Cases with only min_speakers (max 0) take it from the unbounded search (one more or
several more clusters than its best hypothesis holds); for the small and the toy model there is one case where the
bound changes the chosen rank and one where no final hypothesis meets it (the fallback to rank 0), both asserted.
The toy-model cases run at look_ahead 1, so that the tensor-core, cluster and stationary-weights kernels decode them
too.  Only this fixture is written.

Needs the reference checkout (default /root/reference, see oracle/make_golden.py); no GPU.
Usage:  python tools/make_speaker_bounds_golden.py [--jobs 8]
"""
import argparse
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'oracle'))
import make_golden as mg  # noqa: E402  (puts the reference package on sys.path)
import numpy as np  # noqa: E402
import torch  # noqa: E402

# name, model fixture, seed, frames, speakers, (beam, look_ahead, test_iteration), max_speakers, min_speakers
# min_speakers < 0: |value| clusters more than the unbounded search's best hypothesis holds
CASES = [
    ('s_b10_la1_t2', 'model_small.npz', 6201, 60, 5, (10, 1, 2), 3, 0),
    ('s_b1_la1_t1', 'model_small.npz', 6202, 60, 5, (1, 1, 1), 2, 0),
    ('s_b30_la1_t2', 'model_small.npz', 6204, 60, 4, (30, 1, 2), 3, 0),
    ('s_b10_la2_t1', 'model_small.npz', 6205, 40, 5, (10, 2, 1), 2, 0),
    ('s_b30_la2_t2', 'model_small.npz', 6221, 30, 5, (30, 2, 2), 2, 0),
    ('s_b10_la3_t1', 'model_small.npz', 6208, 24, 5, (10, 3, 1), 2, 0),
    ('s_b1_la3_t2', 'model_small.npz', 6216, 24, 5, (1, 3, 2), 2, 0),
    ('s_min_pick', 'model_small.npz', 6210, 60, 5, (10, 1, 1), 0, -1),
    ('s_min_fallback', 'model_small.npz', 6211, 40, 5, (10, 2, 1), 0, -5),
    ('d2_b10_la1_t2', 'model_small_d2.npz', 6301, 50, 5, (10, 1, 2), 2, 0),
    ('d2_b5_la2_t1', 'model_small_d2.npz', 6302, 30, 5, (5, 2, 1), 2, 0),
    ('toy_b10_la1_t2', 'model_toy100.npz', 6401, 60, 5, (10, 1, 2), 2, 0),
    ('toy_b10_la2_t1', 'model_toy100.npz', 6402, 40, 5, (10, 2, 1), 2, 0),
    ('toy_min_pick', 'model_toy100.npz', 6403, 40, 5, (10, 1, 2), 0, -1),
    ('toy_min_fallback', 'model_toy100.npz', 6404, 40, 5, (10, 1, 1), 0, -6),
]


def case_input(fixture, seed, frames, speakers):
  dim = np.load(os.path.join(mg.GOLD, fixture))['w2'].shape[0]
  noise = 0.059 if dim == 256 else 0.08
  return mg.synth.synth_utt(seed, n_frames=frames, dim=dim, n_spk=speakers, noise=noise)[0]


def bound_scores(model, max_speakers):
  """Wraps model._calculate_score: tuples that would take the hypothesis past max_speakers clusters score +inf."""
  if not max_speakers:
    return
  inner = model._calculate_score

  def bounded(beam_state, look_ahead_seq):
    scores = inner(beam_state, look_ahead_seq)
    for idx in np.argwhere(np.isfinite(scores)):
      state = model._update_beam_state(beam_state, look_ahead_seq, tuple(idx))
      if len(state.mean_set) > max_speakers:
        scores[tuple(idx)] = np.inf
    return scores
  model._calculate_score = bounded


def traced_all_ranks(model, seq, iargs, min_speakers):
  """oracle/make_golden.py traced_predict, keeping every final rank."""
  model.rnn_model.eval()
  n = seq.shape[0]
  tiled = torch.from_numpy(np.tile(seq, (iargs.test_iteration, 1))).float()
  beams = [mg.ref_mod.BeamState()]
  win, score, off, nfinite = [], [], [0], []
  for t in range(0, iargs.test_iteration * n, iargs.look_ahead):
    chunk = tiled[t:t + iargs.look_ahead, :]
    la = chunk.shape[0]
    kmax = max(len(b.mean_set) for b in beams)
    table = np.full([iargs.beam_size] + [kmax + 1 + i for i in range(la)], np.inf)
    for r, b in enumerate(beams):
      s = model._calculate_score(b, chunk)
      table[r] = np.pad(s, [(0, kmax - len(b.mean_set))] * la, 'constant', constant_values=np.inf)
    ranked = np.sort(table, axis=None)
    ranked[ranked == np.inf] = 0
    ranked = np.trim_zeros(ranked)
    order = np.argsort(table, axis=None)
    new_beams = []
    for r in range(min(len(ranked), iargs.beam_size)):
      idx = np.unravel_index(order[r], table.shape)
      new_beams.append(model._update_beam_state(beams[idx[0].item()], chunk, idx[1:]))
      win.append([int(v) for v in idx] + [-1] * (iargs.look_ahead - la))
      score.append(float(new_beams[-1].neg_likelihood))
    off.append(len(win))
    nfinite.append(len(ranked))
    beams = new_beams
  final_k = [len(b.mean_set) for b in beams]
  chosen = next((r for r, k in enumerate(final_k) if k >= min_speakers), 0)
  return {
      'win': np.array(win, dtype=np.int32), 'score': np.array(score, dtype=np.float64),
      'off': np.array(off, dtype=np.int64), 'nfinite': np.array(nfinite, dtype=np.int64),
      'final_scores': np.array([float(b.neg_likelihood) for b in beams], dtype=np.float64),
      'final_k': np.array(final_k, dtype=np.int64),
      'final_traces': np.array([b.trace[-n:] for b in beams], dtype=np.int64).reshape(len(beams), n),
      'chosen': np.int64(chosen),
  }


def run_case(case):
  name, fixture, seed, frames, speakers, (beam, la, ti), max_speakers, min_speakers = case
  torch.set_num_threads(1)
  d = dict(np.load(os.path.join(mg.GOLD, fixture)))
  x = case_input(fixture, seed, frames, speakers)
  _, _, ia = mg.ref_args(beam_size=beam, look_ahead=la, test_iteration=ti)
  free = mg.model_from_dict(d)
  unbounded = np.array(free.predict_single(x, ia), dtype=np.int64)
  if min_speakers < 0:
    min_speakers = traced_all_ranks(free, x, ia, 0)['final_k'][0] - min_speakers
  model = mg.model_from_dict(d)
  bound_scores(model, max_speakers)
  labels = np.array(model.predict_single(x, ia), dtype=np.int64)  # rank 0 of the bounded search
  tr = traced_all_ranks(model, x, ia, min_speakers)
  assert np.array_equal(tr['final_traces'][0], labels), name + ': traced search != predict_single'
  if max_speakers:
    assert unbounded.max() + 1 > max_speakers, name + ': max_speakers does not bind'
    assert tr['final_k'].max() <= max_speakers
  if min_speakers:
    assert tr['final_k'][0] < min_speakers, name + ': min_speakers does not bind'
  out = dict(tr, x=x.astype(np.float32), args=np.array([beam, la, ti]), bounds=np.array([max_speakers, min_speakers]),
             unbounded=unbounded, labels=tr['final_traces'][tr['chosen']], model=np.array(fixture))
  print('%-16s unbounded clusters %d  final_k %s  chosen %d' % (name, unbounded.max() + 1, tr['final_k'].tolist(),
                                                               tr['chosen']), flush=True)
  return name, out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--jobs', type=int, default=8)
  a = ap.parse_args()
  o = {'names': np.array([c[0] for c in CASES])}
  for name, out in mg.pmap(run_case, CASES, a.jobs):
    for k, v in out.items():
      o['{}_{}'.format(name, k)] = v
  for model in ('model_small.npz', 'model_toy100.npz'):  # each model: a min-bound pick and a fallback to rank 0
    picks = [int(o[c[0] + '_chosen']) for c in CASES if c[7] < 0 and c[1] == model]
    assert any(p > 0 for p in picks) and any(p == 0 for p in picks), model + ': need a min-bound pick and a fallback'
  np.savez_compressed(os.path.join(mg.GOLD, 'speaker_bounds_cases.npz'), **o)


if __name__ == '__main__':
  main()
