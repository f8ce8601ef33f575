"""A/B of the look-ahead spill kernel on BASELINE config 3 (toy model, beam 30, look_ahead 2, 132 x 100 frames,
device-resident).  Three legs, each in a process of its own and alternated `--rounds` times:
  new     this build, automatic selection (every tree fits shared memory; the spill launch finds nothing to do)
  force   this build with UISRNN_B200_TREE_SPILL=force (every utterance decoded from the device-memory arena)
  prev    a previous build's library (--prev-lib), for the cost of the always-enqueued spill launch
Each leg prints the median frames/s of --reps timed calls (CUDA events around predict_device); labels must agree
across legs.  The card's name and power limit are printed by the same run.

  python tools/tree_spill_ab.py [--prev-lib PATH] [--rounds 3] [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U, N, BEAM, LA = 132, 100, 30, 2


def worker(reps):
  sys.path.insert(0, ROOT)
  import hashlib
  import numpy as np
  import torch
  from uisrnn_b200 import native
  from uisrnn_b200.synth import synth_utt
  m = native.NativeModel(dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'model_toy100.npz'))))
  xs = np.concatenate([synth_utt(1000 + u, n_frames=N)[0] for u in range(U)]).astype(np.float32)
  x = torch.from_numpy(xs).cuda()
  lab = torch.empty(U * N, dtype=torch.int32, device='cuda')
  off = np.arange(U + 1, dtype=np.int64) * N
  start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  for _ in range(2):  # warm-up
    m.predict_device(x.data_ptr(), off, lab.data_ptr(), beam_size=BEAM, look_ahead=LA)
    m.stats()
  times = []
  for _ in range(reps):
    start.record()
    m.predict_device(x.data_ptr(), off, lab.data_ptr(), beam_size=BEAM, look_ahead=LA)
    stop.record()
    torch.cuda.synchronize()
    times.append(start.elapsed_time(stop) / 1e3)
  st = m.stats()
  t = float(np.median(times))
  print(json.dumps({'fps': U * N / t, 'median_s': t, 'spread': (max(times) - min(times)) / t,
                    'launches': st['kernel_launches'],
                    'labels': hashlib.sha256(lab.cpu().numpy().tobytes()).hexdigest()[:16]}), flush=True)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--prev-lib', default=None)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--reps', type=int, default=5)
  ap.add_argument('--worker', action='store_true')
  a = ap.parse_args()
  if a.worker:
    return worker(a.reps)
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                     capture_output=True, text=True).stdout.strip()
  print('device: %s' % (q or 'n/a'), flush=True)
  legs = [('new', {}), ('force', {'UISRNN_B200_TREE_SPILL': 'force'})]
  if a.prev_lib:
    legs.append(('prev', {'UISRNN_B200_LIB': os.path.abspath(a.prev_lib)}))
  res = {name: [] for name, _ in legs}
  hashes = set()
  for r in range(a.rounds):
    for name, env in legs:
      e = dict(os.environ)
      e.pop('UISRNN_B200_TREE_SPILL', None)
      e.update(env)
      out = subprocess.run([sys.executable, os.path.abspath(__file__), '--worker', '--reps', str(a.reps)], env=e,
                           capture_output=True, text=True, cwd=ROOT)
      if out.returncode != 0:
        sys.exit('%s leg failed:\n%s' % (name, out.stderr[-3000:]))
      d = json.loads(out.stdout.strip().splitlines()[-1])
      res[name].append(d)
      hashes.add(d['labels'])
      print('round %d %-5s %10.0f frames/s  (median of %d: %.4f s, spread %.2f %%, launches %d)' % (
          r, name, d['fps'], a.reps, d['median_s'], 100 * d['spread'], d['launches']), flush=True)
  for name, _ in legs:
    f = sorted(d['fps'] for d in res[name])
    print('%-5s median %10.0f frames/s  range %.0f .. %.0f' % (name, f[len(f) // 2], f[0], f[-1]), flush=True)
  print('labels identical across legs: %s' % (len(hashes) == 1), flush=True)
  if len(hashes) != 1:
    sys.exit(1)


if __name__ == '__main__':
  main()
