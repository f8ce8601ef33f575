"""A/B of speaker bounds on bench.py's workload and on BASELINE config 3, in one run:
  unbounded       this build: toy model, 792 x 500-frame utterances (bench.py's seeds), beam 10, test_iteration 2,
                  host-buffer entry point (what UISRNN.predict calls)
  prev            the same with a previous build (--prev-root: a checkout of it whose library is built)
  max2 / max4     this build, max_speakers 2 / 4 for every utterance
  c3 / c3_max4    config 3 (132 x 100 frames, beam 30, look_ahead 2, device-resident), unbounded / max_speakers 4
  large / prev_large  unbounded (1024, 512) depth-2 look-ahead decode (tools/large_model_probe.py's seeded model,
                  64 x 100 frames, beam 10, look_ahead 2, test_iteration 1, device-resident), this build / the previous
Every leg also reports the work counters of its last call (GRU columns and weight passes per beam step).
Each leg runs in a process of its own, legs alternate for --rounds rounds, and each leg reports the median of --reps
timed calls (host clock around the synchronous call; CUDA events for the device-resident legs).  Labels of
`unbounded` and `prev` must agree.  The card's name and power limit are printed by the same run.

  python tools/speaker_bounds_ab.py [--prev-root DIR] [--rounds 3] [--reps 3]"""
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
LARGE_U, LARGE_N = 64, 100


def worker(root, leg, reps):
  sys.path.insert(0, root)
  import numpy as np
  from uisrnn_b200 import native
  from uisrnn_b200.synth import synth_utt
  assert native.__file__.startswith(root), native.__file__
  if leg == 'large':
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    from large_model_probe import synthetic_model
    m = native.NativeModel(synthetic_model(2))
  else:
    m = native.NativeModel(dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'model_toy100.npz'))))
  bound = {'max2': 2, 'max4': 4, 'c3_max4': 4}.get(leg)
  kw = {} if bound is None else {'max_speakers': bound}
  times = []
  if leg.startswith('c3') or leg == 'large':
    import torch
    if leg == 'large':
      nu, nf, dim, opts = LARGE_U, LARGE_N, 512, dict(beam_size=10, look_ahead=2, test_iteration=1, kcap=32)
      xs = np.concatenate([synth_utt(5000 + u, n_frames=nf, dim=dim, n_spk=4, noise=0.02)[0] for u in range(nu)])
    else:
      nu, nf, opts = C3_U, C3_N, dict(beam_size=30, look_ahead=2)
      xs = np.concatenate([synth_utt(1000 + u, n_frames=nf)[0] for u in range(nu)])
    x = torch.from_numpy(xs.astype(np.float32)).cuda()
    lab = torch.empty(nu * nf, dtype=torch.int32, device='cuda')
    off = np.arange(nu + 1, dtype=np.int64) * nf
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    call = lambda: m.predict_device(x.data_ptr(), off, lab.data_ptr(), **opts, **kw)
    for i in range(reps + 1):
      start.record()
      call()
      stop.record()
      torch.cuda.synchronize()
      if i:
        times.append(start.elapsed_time(stop) / 1e3)
    frames, labels = nu * nf, lab.cpu().numpy()
  else:
    xs = [synth_utt(FIRST_SEED + u, n_frames=BENCH_N)[0] for u in range(BENCH_U)]
    for i in range(reps + 1):
      t0 = time.perf_counter()
      out = m.predict(xs, beam_size=10, look_ahead=1, test_iteration=2, **kw)
      if i:
        times.append(time.perf_counter() - t0)
    frames, labels = BENCH_U * BENCH_N, np.concatenate(out)
  t = float(np.median(times))
  st = m.stats()
  print(json.dumps({'fps': frames / t, 'cols_per_step': st['gru_columns'] / max(st['beam_steps'], 1),
                    'passes_per_step': st['weight_passes'] / max(st['beam_steps'], 1),
                    'median_s': t, 'spread': (max(times) - min(times)) / t,
                    'max_label': int(labels.max()),
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
  legs = [('unbounded', ROOT)] + ([('prev', os.path.abspath(a.prev_root))] if a.prev_root else []) + \
      [('max2', ROOT), ('max4', ROOT), ('c3', ROOT), ('c3_max4', ROOT), ('large', ROOT)] + \
      ([('prev_large', os.path.abspath(a.prev_root))] if a.prev_root else [])
  res = {name: [] for name, _ in legs}
  for r in range(a.rounds):
    for name, root in legs:
      leg = {'prev': 'unbounded', 'prev_large': 'large'}.get(name, name)
      out = subprocess.run([sys.executable, os.path.abspath(__file__), '--worker', leg, '--root', root,
                            '--reps', str(a.reps)], capture_output=True, text=True, cwd=root)
      if out.returncode != 0:
        sys.exit('%s leg failed:\n%s' % (name, out.stderr[-3000:]))
      d = json.loads(out.stdout.strip().splitlines()[-1])
      res[name].append(d)
      print('round %d %-10s %10.0f frames/s  (median of %d: %.4f s, spread %.2f %%, max label %d, labels %s, '
            '%.1f GRU columns / %.2f weight passes per beam step)' % (
                r, name, d['fps'], a.reps, d['median_s'], 100 * d['spread'], d['max_label'], d['labels'],
                d['cols_per_step'], d['passes_per_step']), flush=True)
  for name, _ in legs:
    f = sorted(d['fps'] for d in res[name])
    print('%-10s median %10.0f frames/s  range %.0f .. %.0f' % (name, f[len(f) // 2], f[0], f[-1]), flush=True)
  if a.prev_root:
    same = len({d['labels'] for d in res['unbounded'] + res['prev']}) == 1 and \
        len({d['labels'] for d in res['large'] + res['prev_large']}) == 1
    print('unbounded labels identical to the previous build (both workloads): %s' % same, flush=True)
    if not same:
      sys.exit(1)


if __name__ == '__main__':
  main()
