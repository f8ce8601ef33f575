"""Data-parallel fit() (SURVEY.md 8(e), optional row): sharding a mini-batch over ranks and all-reducing
[un-normalised gradients | loss statistics] gives the single-device iteration.

* `test_shard_export_sum_apply_equals_full_step` runs on ONE GPU: two trainers stand in for two ranks and
  the all-reduce is a torch add -- it pins the C-ABI arithmetic (mode 2 + comm_export + comm_apply).
* `test_fit_nccl_world2` is the real thing (two processes, NCCL); skipped on a box with < 2 GPUs.
* `test_fit_gloo_world3` runs UISRNN.fit in three processes over gloo on one GPU, with a rank that never holds a
  column.
tests/test_gpu_fit_dp_fp64.py pins the same steps per element to float64.
"""
import os
import random
import socket
import sys

import numpy as np
import pytest

from helpers import ROOT

pytestmark = pytest.mark.gpu


def _setup(seed=21, D=64, H=128):
  import torch
  import uisrnn
  from uisrnn_b200 import utils
  from uisrnn_b200.synth import synth_training_set
  np.random.seed(seed); random.seed(seed); torch.manual_seed(seed)
  m, t, _ = uisrnn.parse_arguments([])
  m.observation_dim, m.rnn_hidden_size, m.verbosity = D, H, 0
  t.batch_size, t.learning_rate, t.train_iteration = 13, 1e-3, 12
  seqs, ids = synth_training_set(4100, 30, n_frames=50, dim=D, n_spk=3, noise=0.08)
  return uisrnn, utils, m, t, seqs, ids


def _trainer(model, targs):
  from uisrnn_b200 import native
  state = {k: v.detach().cpu().numpy() for k, v in model.rnn_model.state_dict().items()}
  params = {name: state[name] for name in native.PARAM_ORDER[:8]}
  params['rnn_init_hidden'] = model.rnn_init_hidden.detach().cpu().numpy().reshape(-1)
  params['sigma2'] = model.sigma2.detach().cpu().numpy()
  hp = {'learning_rate': targs.learning_rate, 'sigma_alpha': targs.sigma_alpha, 'sigma_beta': targs.sigma_beta,
        'regularization_weight': targs.regularization_weight, 'grad_max_norm': targs.grad_max_norm,
        'train_sigma2': True}
  return native.NativeTrainer(params, hp, device=0)


def test_shard_export_sum_apply_equals_full_step():
  import torch
  from uisrnn_b200.uisrnn import shard_columns
  uisrnn, utils, m, t, seqs, ids = _setup()
  model = uisrnn.UISRNN(m)
  with torch.no_grad():
    model.rnn_init_hidden.data.normal_(0, 0.1)
    model.sigma2.data.uniform_(0.05, 0.2)
  x, y = utils.concatenate_training_data(seqs, ids, True, True)
  subs, lens = utils.resize_sequence(x, np.array(y), t.num_permutations)
  full = _trainer(model, t)
  world = 3                                     # 13 columns over 3 "ranks": 5 + 4 + 4
  ranks = [_trainer(model, t) for _ in range(world)]
  bufs = [torch.zeros(full.comm_size(), device='cuda') for _ in range(world)]
  for it in range(4):
    rnn_input, lengths = utils.pack_batch(subs, lens, t.batch_size, model.observation_dim)
    want_losses = full.step(rnn_input.astype(np.float32), lengths)
    for r in range(world):
      mine = shard_columns(len(lengths), r, world)
      ll = lengths[mine]
      ranks[r].step_shard(rnn_input[:ll[0], mine, :].astype(np.float32), ll)
      ranks[r].comm_export(bufs[r].data_ptr())
    total = bufs[0] + bufs[1] + bufs[2]
    for r in range(world):
      ranks[r].comm_apply(total.data_ptr())
    want = full.parameters()
    for r in range(world):
      got = ranks[r].parameters()
      got_losses = ranks[r].losses(1)[0]
      assert np.allclose(got_losses, want_losses, rtol=2e-5, atol=1e-6), (it, r, got_losses, want_losses)
      for name in want:
        # one Adam step moves a parameter by <= lr = 1e-3; the shards only re-associate fp32 sums
        assert np.max(np.abs(got[name] - want[name])) < 5e-5, (it, r, name)
    first = ranks[0].parameters()
    for r in range(1, world):
      other = ranks[r].parameters()
      assert all(np.array_equal(first[k], other[k]) for k in first)   # replicas stay bit-identical
  for tr in ranks + [full]:
    tr.close()


def _worker(rank, world, port, out_dir):
  sys.path.insert(0, ROOT)
  sys.path.insert(0, os.path.join(ROOT, 'tests'))
  import torch
  import torch.distributed as dist
  torch.cuda.set_device(rank)
  dist.init_process_group('nccl', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=world,
                          device_id=torch.device('cuda', rank))
  uisrnn, _, m, t, seqs, ids = _setup(seed=21 + 100 * rank)   # ranks start from DIFFERENT weights / RNG
  model = uisrnn.UISRNN(m)
  assert model.device.index == rank
  model.fit(seqs, ids, t)
  out = {k: v.detach().cpu().numpy() for k, v in model.rnn_model.state_dict().items()}
  out['sigma2'] = model.sigma2.detach().cpu().numpy()
  out['h0'] = model.rnn_init_hidden.detach().cpu().numpy()
  out['losses'] = np.array(model.last_training_losses)
  np.savez(os.path.join(out_dir, 'rank%d.npz' % rank), **out)
  dist.destroy_process_group()


def test_fit_nccl_world2(tmp_path):
  import torch
  import torch.multiprocessing as mp
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  with socket.socket() as s:
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
  mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
  a = np.load(str(tmp_path / 'rank0.npz'))
  b = np.load(str(tmp_path / 'rank1.npz'))
  for k in a.files:
    assert np.array_equal(a[k], b[k]), k         # both ranks hold the same model and saw the same losses
  # single-device run from rank 0's start (seed 21)
  uisrnn, _, m, t, seqs, ids = _setup(seed=21)
  model = uisrnn.UISRNN(m)
  model.fit(seqs, ids, t)
  single = {k: v.detach().cpu().numpy() for k, v in model.rnn_model.state_dict().items()}
  assert np.allclose(np.array(model.last_training_losses), a['losses'], rtol=1e-3)
  for k, v in single.items():
    assert np.max(np.abs(v - a[k])) < 2e-4, k     # 12 Adam steps of <= 1e-3 each; fp32 re-association only


GLOO_CONFIGS = {
    # two columns over three ranks: rank 2 holds none in any iteration and only adds zeros and applies the sum
    'ndarray-batch2': dict(batch=2),
    # bfloat16 tensors read in place, two layers with inter-layer dropout (each rank masks its own columns)
    'bf16-depth2-dropout-batch4': dict(batch=4, depth=2, dropout=0.2, tensors=True),
}


def _configure(m, t, config):
  t.batch_size = config['batch']
  m.rnn_depth = config.get('depth', 1)
  m.rnn_dropout = config.get('dropout', 0.0)


def _fit_outputs(model):
  out = {k: v.detach().cpu().numpy() for k, v in model.rnn_model.state_dict().items()}
  out['sigma2'] = model.sigma2.detach().cpu().numpy()
  out['h0'] = model.rnn_init_hidden.detach().cpu().numpy()
  out['losses'] = np.array(model.last_training_losses)
  out['loss_terms'] = np.array(model.last_training_loss_terms)
  return out


def _gloo_worker(rank, world, port, out_dir, config):
  sys.path.insert(0, ROOT)
  sys.path.insert(0, os.path.join(ROOT, 'tests'))
  import torch
  import torch.distributed as dist
  dist.init_process_group('gloo', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=world)
  uisrnn, _, m, t, seqs, ids = _setup(seed=21 + 100 * rank)   # ranks start from DIFFERENT weights / RNG
  _configure(m, t, config)
  model = uisrnn.UISRNN(m)
  if config.get('tensors'):
    seqs = [torch.from_numpy(s).cuda().bfloat16() for s in seqs]
  model.fit(seqs, ids, t)
  assert model.last_fit_backend == 'native'
  np.savez(os.path.join(out_dir, 'rank%d.npz' % rank), **_fit_outputs(model))
  dist.destroy_process_group()


@pytest.mark.parametrize('name', list(GLOO_CONFIGS))
def test_fit_gloo_world3(tmp_path, name):
  """Data-parallel fit() in three processes on one GPU over gloo, mini-batches narrower than or not a multiple of
  the world: every rank ends with the same model, losses and loss terms, bit for bit; without dropout the model is
  the single-process fit from rank 0's start, within the bounds of test_fit_nccl_world2."""
  import torch.multiprocessing as mp
  config = GLOO_CONFIGS[name]
  world = 3
  with socket.socket() as s:
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
  mp.spawn(_gloo_worker, args=(world, port, str(tmp_path), config), nprocs=world, join=True)
  got = [np.load(str(tmp_path / ('rank%d.npz' % r))) for r in range(world)]
  assert len(got[0]['losses']) == 12
  for r in range(1, world):
    for k in got[0].files:
      assert np.array_equal(got[0][k], got[r][k]), (r, k)
  if config.get('dropout'):
    return
  uisrnn, _, m, t, seqs, ids = _setup(seed=21)
  _configure(m, t, config)
  model = uisrnn.UISRNN(m)
  model.fit(seqs, ids, t)
  single = _fit_outputs(model)
  assert np.allclose(single['losses'], got[0]['losses'], rtol=1e-3)
  for k in single:
    if k not in ('losses', 'loss_terms'):
      assert np.max(np.abs(single[k] - got[0][k])) < 2e-4, k
