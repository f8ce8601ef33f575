"""Throughput of score() on bench.py's workload: 792 x 500-frame synth_utt utterances (bench.py's seeds),
model_toy100.npz (hidden 512, dim 256), scored with the TRUE labels synth_utt returns.

Reports, in one run on one GPU (with the card's name and power limit):
  score_device   frames/s of uis_score_device on device-resident inputs (CUDA events, median of --reps warmed calls)
  score_host     frames/s of uis_score from host float64 arrays, end to end (host clock around the synchronous call)
  predict_device frames/s of uis_predict_device on the same list (beam 10, test_iteration 2: bench.py's decode)
  gru_columns, the chain kernel's time (beam_ms) and its useful FP32 rate: 2 * (3 H^2 + H^2 + H D) flops per GRU +
  MLP column (W_hh, W1, W2) over the kernel time, against the FFMA peak at the card's max SM clock (132 SMs x 128 FMA lanes x 2).

  python tools/score_bench.py [--reps 10]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BENCH_U, BENCH_N, FIRST_SEED = 792, 500, 100000


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=10)
  a = ap.parse_args()
  import numpy as np
  import torch
  from uisrnn_b200 import native
  from uisrnn_b200.synth import synth_utt
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader,nounits'],
                     capture_output=True, text=True).stdout.strip().splitlines()[0]
  name, power, clock = [v.strip() for v in q.split(',')]
  m = native.NativeModel(dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'model_toy100.npz'))))
  utts = [synth_utt(FIRST_SEED + u, n_frames=BENCH_N) for u in range(BENCH_U)]
  xs = [u[0] for u in utts]
  from uisrnn_b200.uisrnn import canonical_labels
  labels = [canonical_labels(u[1]) for u in utts]
  frames = BENCH_U * BENCH_N
  off = np.arange(BENCH_U + 1, dtype=np.int64) * BENCH_N
  x_dev = torch.from_numpy(np.concatenate(xs).astype(np.float32)).cuda()
  l_dev = torch.from_numpy(np.concatenate(labels)).cuda()
  s_dev = torch.empty(BENCH_U, dtype=torch.float32, device='cuda')
  lab_dev = torch.empty(frames, dtype=torch.int32, device='cuda')
  ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

  def timed_device(call):
    ts, stats = [], None
    for i in range(a.reps + 2):
      ev0.record()
      call()
      ev1.record()
      torch.cuda.synchronize()
      if i >= 2:
        ts.append(ev0.elapsed_time(ev1) / 1e3)
        stats = m.stats()
    return float(np.median(ts)), stats

  t_dev, st = timed_device(lambda: m.score_device(x_dev.data_ptr(), off, l_dev.data_ptr(), s_dev.data_ptr()))
  host = m.score(xs, labels)
  assert np.array_equal(host.view(np.uint32), s_dev.cpu().numpy().view(np.uint32)), 'host and device entry points differ'
  ts = []
  for i in range(a.reps + 1):
    t0 = time.perf_counter()
    m.score(xs, labels)
    if i:
      ts.append(time.perf_counter() - t0)
  t_host = float(np.median(ts))
  t_pred, _ = timed_device(lambda: m.predict_device(x_dev.data_ptr(), off, lab_dev.data_ptr(), beam_size=10,
                                                    look_ahead=1, test_iteration=2))
  H, D = m.H, m.D
  flops = 2.0 * st['gru_columns'] * (3 * H * H + H * H + H * D)  # W_hh, W1, W2 per column (W_ih x: the prepass)
  kernel_s = st['beam_ms'] / 1e3
  peak = 132 * 128 * 2 * float(clock) * 1e6
  print(json.dumps({
      'device': name, 'power_limit_w': float(power), 'max_sm_clock_mhz': float(clock), 'frames': frames,
      'score_device_fps': frames / t_dev, 'score_host_fps': frames / t_host, 'predict_device_fps': frames / t_pred,
      'gru_columns': st['gru_columns'], 'weight_passes': st['weight_passes'], 'chain_kernel_ms': st['beam_ms'],
      'prepass_ms': st['prepass_ms'], 'chain_kernel_tflops': flops / kernel_s / 1e12,
      'ffma_peak_share': flops / kernel_s / peak, 'max_k': st['max_k']}), flush=True)


if __name__ == '__main__':
  main()
