"""A/B of N-best predict() on bench.py's workload and on BASELINE config 3, in one run:
  plain           this build: toy model, 792 x 500-frame utterances (bench.py's seeds), beam 10, test_iteration 2,
                  host-buffer entry point (what UISRNN.predict calls), no n_best
  prev            the same with a previous build (--prev-root: a checkout of it whose library is built)
  nb10            this build, the same workload with n_best = 10
  c3 / c3_nb10    config 3 (132 x 100 frames, beam 30, look_ahead 2, device-resident), without n_best / n_best = 10
Each leg runs in a process of its own, legs alternate for --rounds rounds, and each leg reports the median of --reps
timed calls (host clock around the synchronous call; CUDA events for the device-resident legs).  Labels of `plain`
and `prev` must agree, and so must plane 0 of `nb10` (of `c3_nb10`) and the labels of `plain` (of `c3`).  The card's
name and power limit are printed by the same run.

  python tools/nbest_ab.py [--prev-root DIR] [--rounds 3] [--reps 3]"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BENCH_U, BENCH_N, FIRST_SEED = 792, 500, 100000
C3_U, C3_N = 132, 100


def worker(root, leg, reps):
  sys.path.insert(0, root)
  import numpy as np
  from uisrnn_b200 import native
  from uisrnn_b200.synth import synth_utt
  assert native.__file__.startswith(root), native.__file__
  m = native.NativeModel(dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'model_toy100.npz'))))
  k = 10 if leg.endswith('nb10') else None
  times = []
  if leg.startswith('c3'):
    import torch
    nu, nf = C3_U, C3_N
    x = torch.from_numpy(np.concatenate([synth_utt(1000 + u, n_frames=nf)[0] for u in range(nu)]).astype(np.float32)).cuda()
    lab = torch.empty((k or 1) * nu * nf, dtype=torch.int32, device='cuda')
    sc = torch.empty(nu * (k or 1), dtype=torch.float32, device='cuda')
    off = np.arange(nu + 1, dtype=np.int64) * nf
    kw = dict(n_best=k, scores_ptr=sc.data_ptr()) if k else {}
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for i in range(reps + 1):
      start.record()
      m.predict_device(x.data_ptr(), off, lab.data_ptr(), beam_size=30, look_ahead=2, **kw)
      stop.record()
      torch.cuda.synchronize()
      if i:
        times.append(start.elapsed_time(stop) / 1e3)
    frames, labels = nu * nf, lab.cpu().numpy()[:nu * nf]
  else:
    xs = [synth_utt(FIRST_SEED + u, n_frames=BENCH_N)[0] for u in range(BENCH_U)]
    for i in range(reps + 1):
      t0 = time.perf_counter()
      out = m.predict(xs, beam_size=10, look_ahead=1, test_iteration=2, **({'n_best': k} if k else {}))
      if i:
        times.append(time.perf_counter() - t0)
    frames, labels = BENCH_U * BENCH_N, np.concatenate([o[0] for o in out[0]] if k else out)
  t = float(np.median(times))
  print(json.dumps({'fps': frames / t, 'median_s': t, 'spread': (max(times) - min(times)) / t,
                    'labels': hashlib.sha256(labels.astype(np.int32).tobytes()).hexdigest()[:16]}), flush=True)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--prev-root', default=None)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--reps', type=int, default=3)
  ap.add_argument('--worker', default=None)
  ap.add_argument('--root', default=ROOT)
  a = ap.parse_args()
  if a.worker:
    return worker(a.root, a.worker, a.reps)
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                     capture_output=True, text=True).stdout.strip()
  print('device: %s' % (q or 'n/a'), flush=True)
  legs = [('plain', ROOT)] + ([('prev', os.path.abspath(a.prev_root))] if a.prev_root else []) + \
      [('nb10', ROOT), ('c3', ROOT), ('c3_nb10', ROOT)]
  res = {name: [] for name, _ in legs}
  for r in range(a.rounds):
    for name, root in legs:
      out = subprocess.run([sys.executable, os.path.abspath(__file__), '--worker', 'plain' if name == 'prev' else name,
                            '--root', root, '--reps', str(a.reps)], capture_output=True, text=True, cwd=root)
      if out.returncode != 0:
        sys.exit('%s leg failed:\n%s' % (name, out.stderr[-3000:]))
      d = json.loads(out.stdout.strip().splitlines()[-1])
      res[name].append(d)
      print('round %d %-8s %10.0f frames/s  (median of %d: %.4f s, spread %.2f %%, labels %s)' % (
          r, name, d['fps'], a.reps, d['median_s'], 100 * d['spread'], d['labels']), flush=True)
  for name, _ in legs:
    f = sorted(d['fps'] for d in res[name])
    print('%-8s median %10.0f frames/s  range %.0f .. %.0f' % (name, f[len(f) // 2], f[0], f[-1]), flush=True)
  same = len({d['labels'] for d in res['plain'] + res['nb10'] + res.get('prev', [])}) == 1 and \
      len({d['labels'] for d in res['c3'] + res['c3_nb10']}) == 1
  print('labels identical across legs (plane 0 for n_best): %s' % same, flush=True)
  if not same:
    sys.exit(1)


if __name__ == '__main__':
  main()
