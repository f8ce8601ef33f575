"""fit() iteration probe (BASELINE config 4 shape: D=256, H=512, 50 k frames): wall-clock and device time per
iteration of the device trainer for batch widths and depths.  One JSON line per case."""
import json, os, random, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from uisrnn_b200 import native, utils
from uisrnn_b200.synth import synth_training_set

iters = int(sys.argv[1]) if len(sys.argv) > 1 else 60
D, H = 256, 512
np.random.seed(0); random.seed(0); torch.manual_seed(0)
seqs, ids = synth_training_set(2000, 500, n_frames=100, dim=D, n_spk=3)
x, y = utils.concatenate_training_data(seqs, ids, True, True)
index_lists, lens = utils.resize_indices(np.array(y), 10)
torch.zeros(1).cuda()


def params(depth):
  rng = np.random.default_rng(1)
  p = {}
  for l in range(depth):
    k = D if l == 0 else H
    p['gru.weight_ih_l%d' % l] = rng.normal(0, 0.05, (3 * H, k)).astype(np.float32)
    p['gru.weight_hh_l%d' % l] = rng.normal(0, 0.05, (3 * H, H)).astype(np.float32)
    p['gru.bias_ih_l%d' % l] = np.zeros(3 * H, np.float32)
    p['gru.bias_hh_l%d' % l] = np.zeros(3 * H, np.float32)
  p['linear_mean1.weight'] = rng.normal(0, 0.05, (H, H)).astype(np.float32); p['linear_mean1.bias'] = np.zeros(H, np.float32)
  p['linear_mean2.weight'] = rng.normal(0, 0.05, (D, H)).astype(np.float32); p['linear_mean2.bias'] = np.zeros(D, np.float32)
  p['rnn_init_hidden'] = np.zeros(depth * H, np.float32); p['sigma2'] = np.full(D, 0.1, np.float32)
  return p


CASES = ((1, 32, 0.0), (1, 64, 0.0), (1, 128, 0.0), (2, 32, 0.2), (1, 8, 0.0), (1, 10, 0.0), (1, 16, 0.0))
if len(sys.argv) > 2 and sys.argv[2] == 'small':
  CASES = CASES[4:]
for depth, batch, dropout in CASES:
  hp = {'learning_rate': 1e-3, 'sigma_alpha': 1.0, 'sigma_beta': 1.0, 'regularization_weight': 1e-5, 'grad_max_norm': 5.0,
        'train_sigma2': True, 'rnn_depth': depth, 'rnn_dropout': dropout, 'dropout_seed': 7}
  tr = native.NativeTrainer(params(depth), hp)
  tr.set_corpus(x, index_lists)
  sampler = utils.BatchSampler(lens, batch)
  np.random.seed(3)
  for _ in range(5):
    tr.step_corpus(sampler.draw()[0])
  tr.losses(1)
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  rows, host = 0, 0.0
  t0 = time.perf_counter()
  e0.record()
  for _ in range(iters):
    h0 = time.perf_counter()
    chosen, li = sampler.draw()
    rows += int(li.sum())
    tr.step_corpus(chosen)
    host += time.perf_counter() - h0
  e1.record()
  last = tr.losses(1)
  wall = time.perf_counter() - t0
  print(json.dumps({'depth': depth, 'batch': batch, 'dropout': dropout, 'iters': iters,
                    'wall_ms_per_it': round(1e3 * wall / iters, 3), 'device_ms_per_it': round(e0.elapsed_time(e1) / iters, 3),
                    'host_enqueue_ms_per_it': round(1e3 * host / iters, 3), 'packed_rows_per_s': round(rows / wall),
                    'loss1_last': float(last[0, 0])}), flush=True)
  tr.close()
