"""The cost of running a list in groups of whole utterances, on bench.py's workload (tools/score_bench.py's 792 x
500-frame synth_utt utterances, bench.py's seeds, model_toy100.npz: hidden 512, dim 256), scored with the TRUE labels.

Three workloads, each at once (no limit) and with UISRNN_B200_MAX_ROWS forcing 4 and 16 groups:
  score_numpy     UISRNN.score of float64 ndarrays with host labels (host clock around the call)
  score_tensor    UISRNN.score of fp32 CUDA tensors with int64 CUDA label tensors (host clock around the call and a
                  torch.cuda.synchronize)
  predict_tensor  UISRNN.predict of fp32 CUDA tensors (host clock: the call synchronises once at its end)
Medians of --reps warmed calls, the limits alternated within every round.  The scores of the grouped calls must equal
the ungrouped ones bit for bit; the predict labels are compared and the share of identical utterances reported (a group
of fewer utterances than SMs may be planned onto a latency-mode kernel, whose scores differ in the last bits, so a
near-tied hypothesis may swap).  Prints one JSON line with the card's name and power limit.

  python tools/group_bench.py [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=5)
  a = ap.parse_args()
  import numpy as np
  import torch
  from score_bench import BENCH_N, BENCH_U, FIRST_SEED
  from helpers import inference_args, load_weights, uisrnn_from_weights
  from uisrnn_b200.synth import synth_utt
  from uisrnn_b200.uisrnn import canonical_labels
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader,nounits'],
                     capture_output=True, text=True).stdout.strip().splitlines()[0]
  name, power = [v.strip() for v in q.split(',')]
  model = uisrnn_from_weights(load_weights('model_toy100.npz'), enable_cuda=True)
  args = inference_args(beam_size=10, look_ahead=1, test_iteration=2)
  utts = [synth_utt(FIRST_SEED + u, n_frames=BENCH_N) for u in range(BENCH_U)]
  xs = [u[0] for u in utts]
  ids = [np.asarray(u[1]) for u in utts]
  frames = BENCH_U * BENCH_N
  ts = [torch.from_numpy(x).float().cuda() for x in xs]
  id_ts = [torch.from_numpy(canonical_labels(i).astype(np.int64) * 7919 - 10 ** 12).cuda() for i in ids]
  native = model._native_model()  # pylint: disable=protected-access
  # (groups, UISRNN_B200_MAX_ROWS): every utterance has BENCH_N frames, so ceil(U / groups) utterances per group
  limits = [(1, None)] + [(g, -(-BENCH_U // g) * BENCH_N) for g in (4, 16)]
  legs = {
      'score_numpy': lambda: model.score(xs, ids),
      'score_tensor': lambda: model.score(ts, id_ts).cpu().numpy(),
      'predict_tensor': lambda: [l.cpu().numpy() for l in model.predict(ts, args)],
  }
  out = {'device': name, 'power_limit_w': float(power), 'frames': frames, 'utterances': BENCH_U, 'reps': a.reps}
  bits = lambda v: np.asarray(v, np.float32).view(np.uint32)
  for leg, call in legs.items():
    times = {g: [] for g, _ in limits}
    results = {}
    for rep in range(a.reps + 1):
      for g, max_rows in limits:
        if max_rows is None:
          os.environ.pop('UISRNN_B200_MAX_ROWS', None)
        else:
          os.environ['UISRNN_B200_MAX_ROWS'] = str(max_rows)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        results[g] = call()
        torch.cuda.synchronize()
        if rep:
          times[g].append(time.perf_counter() - t0)
        got = native.stats()['groups']
        assert got == g, '{}: {} groups, expected {}'.format(leg, got, g)
    os.environ.pop('UISRNN_B200_MAX_ROWS', None)
    for g, _ in limits:
      t = float(np.median(times[g]))
      out['{}_{}g_s'.format(leg, g)] = t
      out['{}_{}g_fps'.format(leg, g)] = frames / t
      if g == 1:
        continue
      out['{}_{}g_overhead_pct'.format(leg, g)] = 100.0 * (t / float(np.median(times[1])) - 1.0)
      if leg.startswith('score'):
        assert np.array_equal(bits(results[g]), bits(results[1])), '{}: {} groups change the scores'.format(leg, g)
        out['{}_{}g_identical'.format(leg, g)] = True
      else:
        same = sum(np.array_equal(x, y) for x, y in zip(results[g], results[1]))
        out['{}_{}g_identical_utterances'.format(leg, g)] = int(same)
  print(json.dumps(out), flush=True)


if __name__ == '__main__':
  main()
