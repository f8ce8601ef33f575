"""predict() and score() from torch CUDA tensors against the other ways in, on bench.py's workload (tools/score_bench.py's
792 x 500-frame synth_utt utterances, bench.py's seeds, model_toy100.npz: hidden 512, dim 256), scored with the TRUE
labels synth_utt returns.

Times, in one run on one GPU (with the card's name and power limit), the median of --reps warmed calls of:
  predict_numpy      UISRNN.predict of float64 ndarrays (host clock around the call)
  predict_tensor     UISRNN.predict of fp32 CUDA tensors (host clock: the call synchronises once at its end)
  predict_device     NativeModel.predict_device on the device-resident fp32 rows (CUDA events)
  score_numpy        UISRNN.score of float64 ndarrays with host labels (host clock)
  score_tensor       UISRNN.score of fp32 CUDA tensors with int64 CUDA label tensors: ids renamed and chains planned on
                     the device (host clock around the call and a torch.cuda.synchronize)
  score_device_sweep NativeModel.score_device_sweep on device rows and canonical labels: the host plan (CUDA events)
and checks that every leg returns the same labels (the predict legs) and the same scores bit for bit (the score legs).

  python tools/tensor_bench.py [--reps 5]"""
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
  labels = [canonical_labels(i) for i in ids]
  frames = BENCH_U * BENCH_N
  off = np.arange(BENCH_U + 1, dtype=np.int64) * BENCH_N
  ts = [torch.from_numpy(x).float().cuda() for x in xs]  # what a GPU embedding model would hand over
  id_ts = [torch.from_numpy(canonical_labels(i).astype(np.int64) * 7919 - 10 ** 12).cuda() for i in ids]
  x_dev = torch.cat(ts)
  l_dev = torch.from_numpy(np.concatenate(labels)).cuda()
  lab_dev = torch.empty(frames, dtype=torch.int32, device='cuda')
  s_dev = torch.empty(BENCH_U, dtype=torch.float32, device='cuda')
  native = model._native_model()  # pylint: disable=protected-access
  ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

  def host_timed(call):
    out, t = None, []
    for i in range(a.reps + 1):
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      out = call()
      torch.cuda.synchronize()
      if i:
        t.append(time.perf_counter() - t0)
    return float(np.median(t)), out

  def event_timed(call):
    t = []
    for i in range(a.reps + 1):
      ev0.record()
      call()
      ev1.record()
      torch.cuda.synchronize()
      if i:
        t.append(ev0.elapsed_time(ev1) / 1e3)
    return float(np.median(t))

  t_pn, lab_n = host_timed(lambda: model.predict(xs, args))
  t_pt, lab_t = host_timed(lambda: model.predict(ts, args))
  t_pd = event_timed(lambda: native.predict_device(x_dev.data_ptr(), off, lab_dev.data_ptr(), beam_size=10,
                                                   look_ahead=1, test_iteration=2))
  flat_n = np.concatenate([np.asarray(l, np.int64) for l in lab_n])
  assert np.array_equal(flat_n, torch.cat(lab_t).cpu().numpy()), 'predict: numpy and tensor labels differ'
  assert np.array_equal(flat_n, lab_dev.cpu().numpy().astype(np.int64)), 'predict: numpy and device labels differ'

  t_sn, sc_n = host_timed(lambda: model.score(xs, ids))
  t_st, sc_t = host_timed(lambda: model.score(ts, id_ts))
  t_sd = event_timed(lambda: native.score_device_sweep(x_dev.data_ptr(), off, l_dev.data_ptr(), s_dev.data_ptr(),
                                                       None))
  bits = lambda v: np.asarray(v, np.float32).view(np.uint32)
  assert np.array_equal(bits(sc_n), bits(sc_t.cpu())), 'score: numpy and tensor scores differ'
  assert np.array_equal(bits(sc_n), bits(s_dev.cpu())), 'score: numpy and device scores differ'
  print(json.dumps({
      'device': name, 'power_limit_w': float(power), 'frames': frames, 'reps': a.reps,
      'predict_numpy_fps': frames / t_pn, 'predict_tensor_fps': frames / t_pt, 'predict_device_fps': frames / t_pd,
      'score_numpy_fps': frames / t_sn, 'score_tensor_fps': frames / t_st, 'score_device_sweep_fps': frames / t_sd,
      'identical': True}), flush=True)


if __name__ == '__main__':
  main()
