"""fit() from training sets already on the GPU against the ndarray route, at the config-4 shape (observation_dim 256,
hidden 512, depth 1, batch 32).  The training set is --utts seeded utterances of --frames frames generated on the GPU
as fp32 embeddings (unit-norm rows around per-utterance speaker centroids), with host string labels.

Legs, in --rounds alternated rounds, each a seeded UISRNN.fit of --iters iterations:
  ndarray   the embeddings' .cpu().double().numpy() inside the timed call, then fit() of the float64 arrays
  fp32      fit() of the fp32 CUDA tensors, read in place by the device trainer
  bf16      fit() of bf16 copies of them (made before the call)
For each leg: the host time from the call to the first enqueued training iteration, the time per iteration over the
iterations after the first --skip (CUDA events on the trainer's stream), and the drop in the device's free memory
between the call and the iteration at --skip (informational: other work shares the card).  It checks that the fp32 and
ndarray legs, and the bf16 leg and an (untimed) ndarray fit of its exact float64 upcast, train the same parameters up
to the run-to-run spread of the trainer (its per-dimension residual sums are float atomics), which it reports as the
largest difference between the ndarray legs of two rounds.  Prints the card's name and power limit with the medians as
one JSON line.

  python tools/fit_tensor_bench.py [--utts 4000] [--frames 500] [--iters 250] [--rounds 2]"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--utts', type=int, default=4000)
  ap.add_argument('--frames', type=int, default=500)
  ap.add_argument('--iters', type=int, default=250)
  ap.add_argument('--skip', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=2)
  a = ap.parse_args()
  import numpy as np
  import torch
  from uisrnn_b200 import arguments, native, uisrnn
  if not torch.cuda.is_available():
    raise SystemExit('fit_tensor_bench needs a CUDA device')
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader,nounits'],
                     capture_output=True, text=True).stdout.strip().splitlines()[0]
  name, power = [v.strip() for v in q.split(',')]
  D, H, n_spk = 256, 512, 4
  gen = torch.Generator(device='cuda').manual_seed(1234)
  host_rng = np.random.default_rng(1234)
  xs, ids = [], []
  for u in range(a.utts):  # runs of ~15 frames per speaker, within-speaker noise as synth.synth_utt
    runs = 1 + host_rng.geometric(1.0 / 15, a.frames)
    spk = np.repeat(host_rng.integers(0, n_spk, len(runs)), runs)[:a.frames]
    centres = torch.randn(n_spk, D, device='cuda', generator=gen)
    centres /= centres.norm(dim=1, keepdim=True)
    x = centres[torch.from_numpy(spk).cuda()] + 0.059 * torch.randn(a.frames, D, device='cuda', generator=gen)
    xs.append((x / x.norm(dim=1, keepdim=True)).float())
    ids.append(['{}_{}'.format(u, s) for s in spk.tolist()])
  xs_bf16 = [x.bfloat16() for x in xs]
  frames = a.utts * a.frames
  m, t, _ = arguments.parse_arguments([])
  m.observation_dim, m.rnn_hidden_size, m.verbosity = D, H, 0
  t.batch_size, t.train_iteration = 32, a.iters
  dev = torch.device('cuda', torch.cuda.current_device())

  step_corpus = native.NativeTrainer.step_corpus
  probe = {}

  def timed_step(self, chosen, mode=0, want_losses=False, stream=0):
    k = probe['steps']
    if k == 0:
      probe['first'] = time.perf_counter()
    if k == a.skip:
      probe['free_at_skip'] = torch.cuda.mem_get_info(dev)[0]
      probe['ev0'].record(torch.cuda.ExternalStream(stream) if stream else torch.cuda.default_stream(dev))
    out = step_corpus(self, chosen, mode, want_losses, stream)
    probe['steps'] = k + 1
    if k + 1 == a.iters:
      probe['ev1'].record(torch.cuda.ExternalStream(stream) if stream else torch.cuda.default_stream(dev))
    return out

  native.NativeTrainer.step_corpus = timed_step

  def run(leg, timed=True):
    np.random.seed(5); random.seed(5); torch.manual_seed(5)
    model = uisrnn.UISRNN(m)
    probe.update(steps=0, ev0=torch.cuda.Event(enable_timing=True), ev1=torch.cuda.Event(enable_timing=True))
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(dev)[0]
    t0 = time.perf_counter()
    if leg == 'ndarray':
      model.fit([x.cpu().double().numpy() for x in xs], ids, t)
    elif leg == 'fp32':
      model.fit(xs, ids, t)
    elif leg == 'bf16':
      model.fit(xs_bf16, ids, t)
    else:  # the ndarray route of the bf16 leg's values
      model.fit([x.double().cpu().numpy() for x in xs_bf16], ids, t)
    torch.cuda.synchronize()
    params = [p.detach().cpu().numpy() for p in model.rnn_model.parameters()] + [
        model.sigma2.detach().cpu().numpy(), model.rnn_init_hidden.detach().cpu().numpy()]
    if not timed:
      return params, None
    return params, {'setup_s': probe['first'] - t0,
                    'iter_ms': probe['ev0'].elapsed_time(probe['ev1']) / (a.iters - a.skip),
                    'free_drop_mb': (free0 - probe['free_at_skip']) / 2 ** 20}

  legs = ('ndarray', 'fp32', 'bf16')
  results = {leg: [] for leg in legs}
  params = {leg: [] for leg in legs}
  run('fp32')  # warm-up: module loads, allocator
  for _ in range(a.rounds):
    for leg in legs:
      p, r = run(leg)
      params[leg].append(p)
      results[leg].append(r)
  bf16_ndarray, _ = run('bf16_ndarray', timed=False)
  diff = lambda p, q: max(float(np.max(np.abs(u - v))) for u, v in zip(p, q))
  out = {'device': name, 'power_limit_w': float(power), 'frames': frames, 'utterances': a.utts, 'iters': a.iters,
         'rounds': a.rounds, 'max_abs_diff_fp32_vs_ndarray': diff(params['fp32'][0], params['ndarray'][0]),
         'max_abs_diff_bf16_vs_upcast_ndarray': diff(params['bf16'][0], bf16_ndarray),
         'max_abs_diff_ndarray_run_to_run': diff(params['ndarray'][0], params['ndarray'][-1])}
  for leg in legs:
    for key in ('setup_s', 'iter_ms', 'free_drop_mb'):
      vals = [r[key] for r in results[leg]]
      out['{}_{}'.format(leg, key)] = float(np.median(vals))
      out['{}_{}_range'.format(leg, key)] = [float(min(vals)), float(max(vals))]
  print(json.dumps(out), flush=True)


if __name__ == '__main__':
  main()
