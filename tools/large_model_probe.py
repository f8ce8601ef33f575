"""Decode throughput of the (hidden 1024, dim 512) kernels: frames/s for 264 x 500-frame utterances on a seeded synthetic
model at rnn_depth 1 / 2 / 4 with look_ahead 1 and at look_ahead 2 and 3 (beam 10) with rnn_depth 1 / 2.  Labels must be
identical across the repeats.  The card's name and power limit are printed by the same run.

The model is untrained; sigma2 = 0.02 keeps its decodes at a handful of clusters per utterance (max_k is printed),
as a trained model's would be: smaller sigma2 makes an untrained model open new clusters all the time."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from uisrnn_b200 import native
from uisrnn_b200.synth import synth_utt

U, N, BEAM, TITER, REPEATS = 264, 500, 10, 2, 3
H, D = 1024, 512


def synthetic_model(depth, seed=1024, sigma2=0.02):
  rng = np.random.default_rng(seed + depth)
  u = lambda *s: (rng.uniform(-1, 1, size=s) / np.sqrt(H)).astype(np.float32)
  w = {'depth': depth, 'w1': u(H, H), 'b1': u(H), 'w2': u(D, H), 'b2': u(D), 'h0': u(depth, 1, H),
       'sigma2': np.full(D, sigma2, np.float32), 'transition_bias': 0.3, 'crp_alpha': 1.0}
  for l in range(depth):
    w['weight_ih_l%d' % l] = u(3 * H, D if l == 0 else H)
    w['weight_hh_l%d' % l] = u(3 * H, H)
    w['bias_ih_l%d' % l] = u(3 * H)
    w['bias_hh_l%d' % l] = u(3 * H)
  return w


def main():
  if not torch.cuda.is_available():
    sys.exit('large_model_probe: no CUDA device')
  query = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
  print('device: %s | nvidia-smi: %s' % (torch.cuda.get_device_name(0), query[0] if query else 'n/a'), flush=True)
  xs = np.concatenate([synth_utt(5000 + u, n_frames=N, dim=D, n_spk=4, mean_run=15, noise=0.02)[0] for u in range(U)])
  x = torch.from_numpy(xs.astype(np.float32)).cuda()
  labels = torch.empty(U * N, dtype=torch.int32, device='cuda')
  off = np.arange(U + 1, dtype=np.int64) * N
  start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  for depth, la in ((1, 1), (2, 1), (4, 1), (1, 2), (2, 2), (1, 3), (2, 3)):
    model = native.NativeModel(synthetic_model(depth))
    kcap, refused = 0, None
    while True:  # grow the cluster tables until the decode fits, as UISRNN.predict does
      try:
        model.predict_device(x.data_ptr(), off, labels.data_ptr(), beam_size=BEAM, look_ahead=la, test_iteration=TITER,
                             kcap=kcap)  # also the warm-up
        torch.cuda.synchronize()
        model.stats()  # an asynchronous call reports the utterances' status here
        break
      except native.NativeError as err:
        if err.code == native.UIS_ERR_CAPACITY:  # a step's look-ahead tree exhausted the spill arena's budget
          refused = str(err)
          break
        if err.code != native.UIS_ERR_OVERFLOW or kcap >= 128:
          raise
        kcap = 32 if kcap == 0 else 2 * kcap
    if refused:
      print('depth %d look_ahead %d beam %d: not timed, %s' % (depth, la, BEAM, refused), flush=True)
      model.close()
      continue
    first = labels.cpu().numpy().copy()
    times = []
    for _ in range(REPEATS):
      start.record()
      model.predict_device(x.data_ptr(), off, labels.data_ptr(), beam_size=BEAM, look_ahead=la, test_iteration=TITER,
                           kcap=kcap)
      stop.record()
      torch.cuda.synchronize()
      times.append(start.elapsed_time(stop) / 1e3)
      assert np.array_equal(labels.cpu().numpy(), first), 'labels differ between repeats'
    st = model.stats()
    t = float(np.median(times))
    print('depth %d look_ahead %d beam %d: %9.0f frames/s (median of %d: %.3f s, spread %.1f %%)  kcap %s max_k %d '
          'weight passes %d ctas %d lanes %d' % (
              depth, la, BEAM, U * N / t, REPEATS, t, 100 * (max(times) - min(times)) / t, kcap or 'default',
              st['max_k'], st['weight_passes'], st['ctas'], st['lanes']), flush=True)
    model.close()


if __name__ == '__main__':
  main()
