"""Why does bench.py's config-4 leg see 5.4 ms per fit() iteration when tools/fit_probe.py sees 2.3 ms on the same
shapes?  Times the same trainer loop before / after the other kernels bench.py runs earlier in the process."""
import json, os, random, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from uisrnn_b200 import native, utils
from uisrnn_b200.synth import synth_training_set, synth_utt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
w = dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'model_toy100.npz')))
np.random.seed(0); random.seed(0)
seqs, ids = synth_training_set(2000, 500, n_frames=100, dim=256, n_spk=3)
xcat, ycat = utils.concatenate_training_data(seqs, ids, True, True)
index_lists, lens = utils.resize_indices(np.array(ycat), 10)
params = {'gru.weight_ih_l0': w['weight_ih_l0'], 'gru.weight_hh_l0': w['weight_hh_l0'], 'gru.bias_ih_l0': w['bias_ih_l0'],
          'gru.bias_hh_l0': w['bias_hh_l0'], 'linear_mean1.weight': w['w1'], 'linear_mean1.bias': w['b1'],
          'linear_mean2.weight': w['w2'], 'linear_mean2.bias': w['b2'], 'rnn_init_hidden': w['h0'].reshape(-1), 'sigma2': w['sigma2']}
hp = {'learning_rate': 1e-3, 'sigma_alpha': 1.0, 'sigma_beta': 1.0, 'regularization_weight': 1e-5, 'grad_max_norm': 5.0, 'train_sigma2': True}
torch.zeros(1).cuda()


def fit_loop(tag, iters=60, seed=0):
  tr = native.NativeTrainer(params, hp)
  tr.set_corpus(xcat, index_lists)
  sampler = utils.BatchSampler(lens, 32)
  np.random.seed(seed)
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  maxl = []
  for i in range(5 + iters):
    if i == 5:
      tr.losses(1); e0.record()
    chosen, li = sampler.draw()
    maxl.append(int(li[0]))
    tr.step_corpus(chosen)
  e1.record()
  last = tr.losses(1)
  print(json.dumps({'when': tag, 'device_ms_per_it': round(e0.elapsed_time(e1) / iters, 3), 'mean_L': float(np.mean(maxl)),
                    'loss1_last': float(last[0, 0])}), flush=True)
  tr.close()


fit_loop('fresh process')
fit_loop('again, other batches', seed=5)
model = native.NativeModel(w)
def predict(U, **kw):
  x = torch.from_numpy(np.concatenate([synth_utt(1000 + u, n_frames=500, dim=256)[0] for u in range(U)]).astype(np.float32)).cuda()
  lab = torch.empty(U * 500, dtype=torch.int32, device='cuda')
  model.predict_device(x.data_ptr(), np.arange(U + 1, dtype=np.int64) * 500, lab.data_ptr(), **kw)
  return model.stats()
predict(264, engine=1); fit_loop('after FFMA beam kernel (U=264)')
predict(1); fit_loop('after cluster beam kernel (U=1)')
predict(300, engine=2); fit_loop('after tensor-core beam kernel (U=300)')
predict(132, beam_size=30, look_ahead=2); fit_loop('after look-ahead tree kernel')
fit_loop('100 iterations', iters=100)
