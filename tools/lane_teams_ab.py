"""A/B of the lane-team selection phases against a previous build, in one run:
  bench       bench.py --gpus 1 --steps K --warmup W in each build's tree: `value` (device-resident, 792 x 500-frame
              utterances, beam 10, 6 lanes per CTA), `e2e` (UISRNN.predict from pinned host arrays) and its secondary
              legs (config 3, config2_U1 = stationary weights, config2_U64, config2_U264_ffma_engine); labels dumped
  beam128     one tensor-core call at beam 128 (132 x 100 frames, kcap 8, max_speakers 8, device-resident, CUDA events)
  tc_bench    tools/tc_bench.py 792 in each build's tree: phase_us_per_cta_step of the tensor-core engine at 6 lanes
Builds alternate for --rounds rounds, each leg in a process of its own.  The card's name and power limit are printed by
the same run; the labels of the two builds must agree.

  python tools/lane_teams_ab.py --prev-root DIR [--rounds 3] [--steps 5] [--warmup 3] [--out DIR]"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def beam128_worker(root, reps):
  sys.path.insert(0, root)
  import torch
  from uisrnn_b200 import native
  from uisrnn_b200.synth import synth_utt
  assert native.__file__.startswith(root), native.__file__
  m = native.NativeModel(dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'model_toy100.npz'))))
  nu, nf = 132, 100
  x = torch.from_numpy(np.concatenate([synth_utt(1000 + u, n_frames=nf)[0] for u in range(nu)]).astype(np.float32)).cuda()
  lab = torch.empty(nu * nf, dtype=torch.int32, device='cuda')
  off = np.arange(nu + 1, dtype=np.int64) * nf
  start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  times = []
  for i in range(reps + 1):
    start.record()
    m.predict_device(x.data_ptr(), off, lab.data_ptr(), beam_size=128, kcap=8, max_speakers=8, engine=2)
    stop.record()
    torch.cuda.synchronize()
    if i:
      times.append(start.elapsed_time(stop))
  st = m.stats()
  assert st['engine'] == 2, st
  print(json.dumps({'ms': float(np.median(times)), 'lanes': st['lanes'],
                    'labels': hashlib.sha256(lab.cpu().numpy().tobytes()).hexdigest()[:16]}), flush=True)


def run(cmd, cwd):
  out = subprocess.run(cmd, capture_output=True, text=True, cwd=cwd)
  if out.returncode != 0:
    sys.exit('%s failed in %s:\n%s' % (' '.join(cmd), cwd, out.stderr[-3000:]))
  return out.stdout


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--prev-root', help='tree of the previous build, its library built')
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--steps', type=int, default=5)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--reps', type=int, default=3)
  ap.add_argument('--out', default=None, help='directory for the dumped labels (default: a new temporary one)')
  ap.add_argument('--beam128-worker', default=None)
  a = ap.parse_args()
  if a.beam128_worker:
    return beam128_worker(a.beam128_worker, a.reps)
  if not a.prev_root:
    ap.error('--prev-root is required')
  out_dir = a.out or tempfile.mkdtemp(prefix='lane_teams_ab_')
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                     capture_output=True, text=True).stdout.strip()
  print('device: %s' % (q or 'n/a'), flush=True)
  builds = [('this', ROOT), ('prev', os.path.abspath(a.prev_root))]
  legs = ['value', 'e2e', 'config3_beam30_lookahead2', 'config2_U1', 'config2_U64', 'config2_U264_ffma_engine',
          'beam128_ms']
  res = {b: {k: [] for k in legs} for b, _ in builds}
  labels = {b: set() for b, _ in builds}
  for r in range(a.rounds):
    for name, root in builds:
      dump = os.path.join(out_dir, '%s_r%d' % (name, r))
      line = run([sys.executable, 'bench.py', '--gpus', '1', '--steps', str(a.steps), '--warmup', str(a.warmup),
                  '--no-cpu-baseline', '--dump-outputs', dump], root).strip().splitlines()[-1]
      d = json.loads(line)
      sec = d.get('secondary', {})
      res[name]['value'].append(d['value'])
      res[name]['e2e'].append(d['e2e']['value'])
      for k in legs[2:6]:
        res[name][k].append(sec.get(k, {}).get('frames_per_s'))
      labels[name].add(hashlib.sha256(np.load(os.path.join(dump, 'labels.npy')).tobytes()).hexdigest()[:16])
      b = json.loads(run([sys.executable, os.path.abspath(__file__), '--beam128-worker', root, '--reps', str(a.reps)],
                         root).strip().splitlines()[-1])
      res[name]['beam128_ms'].append(b['ms'])
      labels[name].add('beam128:' + b['labels'])
      print('round %d %-5s value %.0f  e2e %s  c3 %s  U1 %s  U64 %s  ffma %s  beam128 %.2f ms' % (
          r, name, d['value'], res[name]['e2e'][-1], *[res[name][k][-1] for k in legs[2:6]], b['ms']), flush=True)
  for name, _ in builds:
    for k in legs:
      v = sorted(x for x in res[name][k] if x is not None)
      if v:
        print('%-5s %-26s median %12.2f  range %.2f .. %.2f' % (name, k, v[len(v) // 2], v[0], v[-1]), flush=True)
  for k in legs:
    t = sorted(x for x in res['this'][k] if x is not None)
    p = sorted(x for x in res['prev'][k] if x is not None)
    if t and p:
      print('ratio this/prev %-26s %.4f' % (k, t[len(t) // 2] / p[len(p) // 2]), flush=True)
  same = labels['this'] == labels['prev']
  print('labels identical between builds (bench dump, beam 128): %s' % same, flush=True)
  for name, root in builds:
    print('tc_bench 792 (%s):' % name, flush=True)
    print(run([sys.executable, 'tools/tc_bench.py', '792'], root).strip(), flush=True)
  if not same:
    sys.exit(1)


if __name__ == '__main__':
  main()
