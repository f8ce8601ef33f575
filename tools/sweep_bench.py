"""Decoding-parameter sweep against the per-pair loop it replaces, on a dev-set-sized list: the reference's toy model
(hidden 512, dim 256), 100 synthetic 500-frame utterances, beam 10, test_iteration 2, 16 (crp_alpha, transition_bias)
pairs (4 x 4).  Times, as medians of --reps calls after one warm-up each:
  sweep        one UISRNN.predict(decode_params=pairs) call
  loop         16 predict() calls with model.crp_alpha / transition_bias set before each (the device model is rebuilt)
  loop_engine  the loop on NativeModels created per pair, with the engine / lanes forced to the sweep's plan; its labels
               must equal the sweep's bit for bit
  score        score(decode_params=pairs) of the true labels against 16 per-pair score() calls
Rates are decoded frames per second (U * C * N over wall time).  The card's name and power limit are read by the same
run.  The agreement of the auto-plan loop with the sweep may differ only in near-ties (different engines).

  python tools/sweep_bench.py [--utts 100] [--frames 500] [--reps 3] [--out FILE.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def card():
  out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
  return out


def timed(fn, reps):
  fn()  # warm-up
  ts = []
  for _ in range(reps):
    t0 = time.perf_counter()
    out = fn()
    ts.append(time.perf_counter() - t0)
  return statistics.median(ts), ts, out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--utts', type=int, default=100)
  ap.add_argument('--frames', type=int, default=500)
  ap.add_argument('--reps', type=int, default=3)
  ap.add_argument('--out', default=None)
  a = ap.parse_args()
  import torch
  from helpers import inference_args, load_weights, uisrnn_from_weights
  from uisrnn_b200 import native
  from uisrnn_b200.synth import synth_utt
  assert torch.cuda.is_available(), 'sweep_bench measures the GPU: no CUDA device'
  w = load_weights('model_toy100.npz')
  data = [synth_utt(7000 + i, n_frames=a.frames) for i in range(a.utts)]
  xs, truth = [d[0] for d in data], [list(d[1]) for d in data]
  pairs = [(al, p0) for al in (0.1, 0.5, 1.0, 4.0) for p0 in (0.01, 0.05, 0.2, 0.5)]
  args = inference_args(beam_size=10, test_iteration=2)
  model = uisrnn_from_weights(w, enable_cuda=True)
  frames = a.utts * a.frames * len(pairs)
  res = {'card': card(), 'utterances': a.utts, 'frames': a.frames, 'pairs': len(pairs), 'beam_size': 10,
         'test_iteration': 2}

  t, ts, sweep = timed(lambda: model.predict(xs, args, decode_params=pairs), a.reps)
  st = model._native_model().stats()  # pylint: disable=protected-access
  res['sweep'] = {'s': t, 'all_s': ts, 'frames_per_s': frames / t, 'engine': st['engine'], 'lanes': st['lanes'],
                  'ctas': st['ctas'], 'cluster': st['cluster']}

  def loop():
    out = []
    for al, p0 in pairs:
      model.crp_alpha, model.transition_bias = al, p0
      out.append(model.predict(xs, args))
    model.crp_alpha, model.transition_bias = float(w['crp_alpha']), float(w['transition_bias'])
    return out
  t, ts, looped = timed(loop, a.reps)
  same = sum(g == s for c in range(len(pairs)) for g, s in zip(looped[c], sweep[c]))
  res['loop'] = {'s': t, 'all_s': ts, 'frames_per_s': frames / t,
                 'utterances_equal_to_sweep': '{}/{}'.format(same, a.utts * len(pairs))}

  forced = dict(engine=st['engine'], lanes=st['lanes'], cluster=-1 if st['cluster'] <= 1 else st['cluster'])
  per_pair = []
  for al, p0 in pairs:
    wp = dict(w)
    wp['crp_alpha'], wp['transition_bias'] = al, p0
    per_pair.append(native.NativeModel(wp))
  t, ts, forced_out = timed(lambda: [m.predict(xs, beam_size=10, look_ahead=1, test_iteration=2, **forced)
                                     for m in per_pair], a.reps)
  res['loop_engine'] = {'s': t, 'all_s': ts, 'frames_per_s': frames / t, 'forced': forced}
  for c in range(len(pairs)):
    for u in range(a.utts):
      assert forced_out[c][u].tolist() == sweep[c][u], ('forced-engine loop differs from the sweep', pairs[c], u)
  res['loop_engine']['labels_equal_to_sweep'] = True

  t, ts, scored = timed(lambda: model.score(xs, truth, decode_params=pairs), a.reps)
  res['score_sweep'] = {'s': t, 'all_s': ts, 'frames_per_s': frames / t}
  def score_loop():
    out = []
    for al, p0 in pairs:
      model.crp_alpha, model.transition_bias = al, p0
      out.append(model.score(xs, truth))
    model.crp_alpha, model.transition_bias = float(w['crp_alpha']), float(w['transition_bias'])
    return out
  t, ts, scored_loop = timed(score_loop, a.reps)
  assert scored_loop == scored, 'score sweep differs from the per-pair score() calls'
  res['score_loop'] = {'s': t, 'all_s': ts, 'frames_per_s': frames / t}
  from uisrnn_b200 import evals
  acc = [float(np.mean([evals.compute_sequence_match_accuracy(truth[u], sweep[c][u]) for u in range(a.utts)]))
         for c in range(len(pairs))]
  best = int(np.argmax(acc))
  res['accuracy'] = {'best_pair': pairs[best], 'best': acc[best]}
  line = json.dumps(res)
  print(line)
  if a.out:
    with open(a.out, 'w') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
