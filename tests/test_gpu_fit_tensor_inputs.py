"""fit() from CUDA tensors: every case fits the same seeded training set once from float64 ndarrays and once from
tensors.  The device trainer reads the tensors' rows in place, in their dtype, and gathers the same fp32 batches as
from the ndarrays: the gradients of a step (all but sigma2's) are equal bit for bit.  The trainer sums the squared
residuals per dimension with float atomics across batch columns, so the loss values, the sigma2 gradient and through
them the trained model vary in their last bits from run to run on either path; whole fits are compared to that
spread, and transition_bias (a host computation) exactly."""
import os
import random
import socket
import sys

import numpy as np
import pytest

from helpers import ROOT

pytestmark = pytest.mark.gpu

DTYPES = ('float32', 'float16', 'bfloat16', 'float64')
LAYOUTS = ('contiguous', 'row_strided', 'odd_offset', 'transposed')


def _args(D=32, H=64, depth=1, dropout=0.0, batch=16, iters=6, **training):
  import uisrnn
  m, t, _ = uisrnn.parse_arguments([])
  m.observation_dim, m.rnn_hidden_size, m.rnn_depth, m.rnn_dropout, m.verbosity = D, H, depth, dropout, 0
  t.batch_size, t.learning_rate, t.train_iteration = batch, 1e-3, iters
  for key, value in training.items():
    setattr(t, key, value)
  return m, t


def _data(D=32, n_utt=10, n_frames=40, seed=4700):
  """float64 sequences and their integer speaker labels."""
  from uisrnn_b200.synth import synth_utt
  seqs, ints = [], []
  for u in range(n_utt):
    x, lab = synth_utt(seed + u, n_frames=n_frames - 3 * (u % 4), dim=D, n_spk=3, noise=0.08)
    seqs.append(x)
    ints.append(lab - 2 + 10 * u)  # negative ids too, and distinct speakers per utterance
  return seqs, ints


def _str_ids(ints):
  return [[str(v) for v in lab.tolist()] for lab in ints]


def _to_tensor(a, dtype, layout):
  """A CUDA tensor of dtype holding a's values (rounded to dtype) in the given memory layout."""
  import torch
  t = torch.from_numpy(a).cuda().to(getattr(torch, dtype))
  n, d = t.shape
  if layout == 'contiguous':
    return t
  if layout == 'row_strided':  # rows of a wider tensor
    wide = torch.full((n, d + 6), float('nan'), dtype=t.dtype, device=t.device)
    wide[:, 2:2 + d] = t
    return wide[:, 2:2 + d]
  if layout == 'odd_offset':  # a contiguous view starting at an odd element
    flat = torch.full((1 + n * d,), float('nan'), dtype=t.dtype, device=t.device)
    flat[1:] = t.reshape(-1)
    view = flat[1:].view(n, d)
    assert view.data_ptr() % (2 * t.element_size()) != 0
    return view
  assert layout == 'transposed'  # element stride n
  return t.t().contiguous().t()


def _upcast(tensors):
  """The exact float64 values of tensors, as host ndarrays."""
  import torch
  return [t.to(torch.float64).cpu().numpy() for t in tensors]


def _state(model):
  out = {k: v.detach().cpu().numpy() for k, v in model.rnn_model.state_dict().items()}
  out['sigma2'] = model.sigma2.detach().cpu().numpy()
  out['rnn_init_hidden'] = model.rnn_init_hidden.detach().cpu().numpy()
  out['transition_bias'] = np.array([model.transition_bias, model.transition_bias_denominator])
  out['losses'] = np.array(model.last_training_losses)
  out['loss_terms'] = np.array(model.last_training_loss_terms)
  return out


def _fit(m, t, seqs, ids, calls=1, seed=7, method='fit'):
  import torch
  import uisrnn
  np.random.seed(seed); random.seed(seed); torch.manual_seed(seed)
  model = uisrnn.UISRNN(m)
  for _ in range(calls):
    getattr(model, method)(seqs, ids, t)
  assert model.last_fit_backend == 'native'
  return _state(model)


def _assert_same(want, got):
  """Equal up to the run-to-run spread of the trainer's atomic loss sums (a few fp32 ulps per step, over at most a
  few Adam steps of <= 1e-3 each)."""
  assert want.keys() == got.keys()
  assert len(want['losses']) > 0
  for k in want:
    if k == 'transition_bias':
      assert np.array_equal(want[k], got[k]), k
    else:
      assert want[k].shape == got[k].shape and np.allclose(want[k], got[k], rtol=1e-5, atol=1e-6), k


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('layout', LAYOUTS)
def test_dtypes_and_layouts_match_the_ndarray_fit(dtype, layout):
  m, t = _args()
  seqs, ints = _data()
  ids = _str_ids(ints)
  tensors = [_to_tensor(a, dtype, layout) for a in seqs]
  want = _fit(m, t, _upcast(tensors), ids)
  _assert_same(want, _fit(m, t, tensors, ids))
  # the conversion itself, exactly: the gradients of steps gathered from the rows in place
  import torch
  import uisrnn
  from uisrnn_b200 import utils
  _, y = utils.concatenate_training_data(_upcast(tensors), ids, False, False)
  index_lists, lens = utils.resize_indices(np.array(y), t.num_permutations)
  np.random.seed(3); torch.manual_seed(3)
  _assert_same_steps(uisrnn.UISRNN(m), t, tensors, index_lists, lens)


@pytest.mark.parametrize('config', [
    dict(depth=2, dropout=0.2, batch=48),     # more than one 32-column group
    dict(batch=None),
    dict(num_permutations=1),
    dict(enforce_cluster_id_uniqueness=False),
    dict(D=256, H=512, batch=32, iters=3),    # the default shape
    dict(D=64, H=640, batch=8, iters=3),      # per-step recurrence launches
])
def test_configurations_match_the_ndarray_fit(config):
  import torch
  D = config.pop('D', 32)
  m, t = _args(D=D, **config)
  seqs, ints = _data(D=D, n_utt=12)
  ids = _str_ids(ints)
  tensors = [torch.from_numpy(a).cuda().float() for a in seqs]
  want = _fit(m, t, _upcast(tensors), ids)
  _assert_same(want, _fit(m, t, tensors, ids))


def test_integer_label_tensors_are_their_strings():
  """int32 / int64 label tensors (negative values, strided) train as the str(v) labels; so does a list mixing them
  with host labels."""
  import torch
  m, t = _args()
  seqs, ints = _data()
  tensors = [torch.from_numpy(a).cuda() for a in seqs]
  want = _fit(m, t, seqs, _str_ids(ints))
  labels = []
  for u, lab in enumerate(ints):
    dtype = torch.int32 if u % 2 else torch.int64
    pair = torch.from_numpy(np.stack([lab, lab], 1)).cuda().to(dtype)
    labels.append(pair[:, 1] if u % 3 else pair.t().contiguous()[0])
  _assert_same(want, _fit(m, t, tensors, labels))
  mixed = [labels[u] if u % 2 else _str_ids(ints)[u] for u in range(len(ints))]
  _assert_same(want, _fit(m, t, tensors, mixed))
  with_host_ints = [labels[u] if u % 2 else np.array(_str_ids(ints)[u]) for u in range(len(ints))]
  _assert_same(want, _fit(m, t, tensors, with_host_ints))


def test_single_tensor_forms():
  import torch
  m, t = _args()
  seqs, ints = _data(n_utt=6)
  x = np.concatenate(seqs)
  lab = np.concatenate(ints)
  xt = torch.from_numpy(x).cuda().half()
  xh = xt.double().cpu().numpy()
  want = _fit(m, t, xh, [str(v) for v in lab.tolist()])
  _assert_same(want, _fit(m, t, xt, torch.from_numpy(lab).cuda()))
  want = _fit(m, t, xh, np.array([str(v) for v in lab.tolist()]), method='fit_concatenated')
  _assert_same(want, _fit(m, t, xt, torch.from_numpy(lab).cuda(), method='fit_concatenated'))
  _assert_same(want, _fit(m, t, xt, [str(v) for v in lab.tolist()], method='fit_concatenated'))


def test_successive_fits_average_the_transition_bias():
  import torch
  m, t = _args()
  seqs, ints = _data()
  tensors = [torch.from_numpy(a).cuda().bfloat16() for a in seqs]
  want = _fit(m, t, _upcast(tensors), _str_ids(ints), calls=2)
  got = _fit(m, t, tensors, [torch.from_numpy(v).cuda() for v in ints], calls=2)
  _assert_same(want, got)


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


def _assert_same_gradients(want, got):
  """Gradients of one step: bit for bit, except sigma2's, which takes the trainer's atomic residual sums."""
  assert want.keys() == got.keys()
  for k in want:
    assert np.array_equal(want[k], got[k]) if k != 'sigma2' else np.allclose(want[k], got[k], rtol=1e-5), k


def _assert_same_steps(model, t, tensors, index_lists, lens, draws=2):
  """step_corpus(mode=1) on `tensors` read in place against the float64 corpus of their exact values."""
  from uisrnn_b200 import utils
  tr, ref = _trainer(model, t), _trainer(model, t)
  tr.set_corpus_device(tensors, index_lists)
  ref.set_corpus(np.concatenate(_upcast(tensors)), index_lists)
  sampler = utils.BatchSampler(lens, t.batch_size)
  for _ in range(draws):
    chosen, _ = sampler.draw()
    tr.step_corpus(chosen, mode=1)
    ref.step_corpus(chosen, mode=1)
    _assert_same_gradients(ref.gradients(), tr.gradients())
  tr.close()
  ref.close()


def _corpus(seed=3):
  import torch
  import uisrnn
  from uisrnn_b200 import utils
  np.random.seed(seed); random.seed(seed); torch.manual_seed(seed)
  m, t = _args(batch=13)
  seqs, ints = _data()
  x, y = utils.concatenate_training_data(seqs, _str_ids(ints), True, True)
  index_lists, lens = utils.resize_indices(np.array(y), t.num_permutations)
  return uisrnn.UISRNN(m), t, x, index_lists, lens


def test_trainer_reads_the_rows_in_place():
  """Rows overwritten after set_corpus_device are what the next step gathers."""
  import torch
  from uisrnn_b200 import utils
  model, t, x, index_lists, lens = _corpus()
  rows = torch.from_numpy(x).cuda().float()
  tr = _trainer(model, t)
  tr.set_corpus_device([rows[:50], rows[50:]], index_lists)
  chosen, _ = utils.BatchSampler(lens, t.batch_size).draw()
  rows[::3] = torch.randn_like(rows[::3])
  tr.step_corpus(chosen, mode=1)
  ref = _trainer(model, t)
  ref.set_corpus(rows.double().cpu().numpy(), index_lists)
  ref.step_corpus(chosen, mode=1)
  _assert_same_gradients(ref.gradients(), tr.gradients())
  tr.close()
  ref.close()


def test_steps_run_on_the_given_stream():
  """Rows filled on a non-blocking side stream behind a delay: set_corpus_device and step_corpus enqueued on that stream
  read them after the fill, without the host waiting for it.  A step on any other stream would read the zeros."""
  import torch
  from uisrnn_b200 import utils
  model, t, x, index_lists, lens = _corpus()
  src = torch.from_numpy(x).cuda().float()
  chosen, _ = utils.BatchSampler(lens, t.batch_size).draw()
  ref = _trainer(model, t)
  ref.set_corpus(src.double().cpu().numpy(), index_lists)
  ref.step_corpus(chosen, mode=1)
  want = ref.gradients()
  ref.close()
  tr = _trainer(model, t)
  torch.cuda.synchronize()
  side = torch.cuda.Stream()
  with torch.cuda.stream(side):
    rows = torch.zeros_like(src)
    torch.cuda._sleep(500_000_000)  # pylint: disable=protected-access
    rows.copy_(src)
    tr.set_corpus_device([rows[:50], rows[50:]], index_lists, stream=side.cuda_stream)
    tr.step_corpus(chosen, mode=1, stream=side.cuda_stream)
  _assert_same_gradients(want, tr.gradients())
  tr.close()


def test_shard_export_sum_apply_equals_full_step_from_tensors():
  """The one-GPU stand-in of a data-parallel step with tensor corpora: mode 2 + comm_export, a torch sum and
  comm_apply equal the full step; the full step from tensors equals the one from the float64 corpus bit for bit."""
  import torch
  from uisrnn_b200 import utils
  from uisrnn_b200.uisrnn import shard_columns
  model, t, x, index_lists, lens = _corpus(seed=5)
  rows = torch.from_numpy(x).cuda().half()
  xh = rows.double().cpu().numpy()
  full, host = _trainer(model, t), _trainer(model, t)
  full.set_corpus_device([rows], index_lists)
  host.set_corpus(xh, index_lists)
  world = 3
  ranks = [_trainer(model, t) for _ in range(world)]
  for r in ranks:
    r.set_corpus_device([rows[:70], rows[70:]], index_lists)
  bufs = [torch.zeros(full.comm_size(), device='cuda') for _ in range(world)]
  sampler = utils.BatchSampler(lens, t.batch_size)
  for it in range(3):
    chosen, _ = sampler.draw()
    full.step_corpus(chosen)
    host.step_corpus(chosen)
    for r in range(world):
      ranks[r].step_corpus(chosen[shard_columns(len(chosen), r, world)], mode=2)
      ranks[r].comm_export(bufs[r].data_ptr())
    torch.cuda.synchronize()
    total = bufs[0] + bufs[1] + bufs[2]
    torch.cuda.synchronize()
    for r in range(world):
      ranks[r].comm_apply(total.data_ptr())
    want = full.parameters()
    exact = host.parameters()
    assert all(np.allclose(want[k], exact[k], rtol=1e-5, atol=1e-7) for k in want), it
    for r in range(world):
      got = ranks[r].parameters()
      for name in want:
        assert np.max(np.abs(got[name] - want[name])) < 5e-5, (it, r, name)
  for tr in ranks + [full, host]:
    tr.close()


def _worker(rank, world, port, out_dir):
  sys.path.insert(0, ROOT)
  sys.path.insert(0, os.path.join(ROOT, 'tests'))
  import torch
  import torch.distributed as dist
  torch.cuda.set_device(rank)
  dist.init_process_group('nccl', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=world,
                          device_id=torch.device('cuda', rank))
  m, t = _args(batch=13, iters=8)
  seqs, ints = _data()
  tensors = [torch.from_numpy(a).cuda().float() for a in seqs]
  out = {}
  for leg, (xs, ids) in (('ndarray', (_upcast(tensors), _str_ids(ints))),
                         ('tensor', (tensors, [torch.from_numpy(v).cuda() for v in ints]))):
    state = _fit(m, t, xs, ids, seed=21 + 100 * rank)  # ranks start from different weights and RNG states
    out.update({leg + '/' + k: v for k, v in state.items()})
  np.savez(os.path.join(out_dir, 'rank%d.npz' % rank), **out)
  dist.destroy_process_group()


def test_fit_nccl_world2_from_tensors_equals_ndarrays(tmp_path):
  import torch
  import torch.multiprocessing as mp
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  with socket.socket() as s:
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
  mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
  for rank in range(2):
    got = np.load(str(tmp_path / ('rank%d.npz' % rank)))
    keys = [k.split('/', 1)[1] for k in got.files if k.startswith('ndarray/')]
    for k in keys:
      a, b = got['ndarray/' + k], got['tensor/' + k]
      assert np.array_equal(a, b) if k == 'transition_bias' else np.allclose(a, b, rtol=1e-5, atol=1e-6), (rank, k)


def test_errors():
  import torch
  import uisrnn
  m, t = _args()
  model = uisrnn.UISRNN(m)
  seqs, ints = _data(n_utt=3)
  x = [torch.from_numpy(a).cuda() for a in seqs]
  ids = _str_ids(ints)
  with pytest.raises(TypeError, match='train_sequences must be all numpy arrays or all torch tensors'):
    model.fit([x[0], seqs[1], x[2]], ids, t)
  with pytest.raises(TypeError, match='share a dtype'):
    model.fit([x[0], x[1].float(), x[2]], ids, t)
  with pytest.raises(TypeError, match='float32, float16, bfloat16 or float64'):
    model.fit([v.int() for v in x], ids, t)
  with pytest.raises(ValueError, match="train_sequence tensors must be on the model's device"):
    model.fit([x[0], x[1].cpu(), x[2]], ids, t)
  with pytest.raises(ValueError, match='train_sequence does not match the dimension'):
    model.fit([v[:, :-1] for v in x], ids, t)
  with pytest.raises(ValueError, match='train_sequence must be 2-dim array'):
    model.fit([x[0][0], x[1], x[2]], ids, t)
  with pytest.raises(ValueError, match='train_sequence must be 2-dim array'):
    model.fit_concatenated(x[0][0], ids[0][:1], t)
  with pytest.raises(TypeError, match='integer dtype'):
    model.fit(x, [torch.from_numpy(ints[0]).cuda().float()] + ids[1:], t)
  with pytest.raises(ValueError, match='labels for'):
    model.fit(x, [torch.from_numpy(ints[0][:-1]).cuda()] + ids[1:], t)
  with pytest.raises(ValueError, match='label tensor is on'):
    model.fit(x, [torch.from_numpy(ints[0])] + ids[1:], t)
  with pytest.raises(ValueError, match='train_sequence length is not equal'):
    model.fit_concatenated(x[0], ids[0][:-1], t)
  with pytest.raises(TypeError, match='numpy array of strings'):
    model.fit_concatenated(x[0], [int(v) for v in ints[0]], t)
  assert model.transition_bias is None  # no error got as far as the estimate
  with pytest.raises(ValueError, match='same length'):  # (a host label sequence is checked where ndarrays' are)
    model.fit(x, [ids[0][:-1]] + ids[1:], t)
  m5, t5 = _args(depth=5)
  deep = uisrnn.UISRNN(m5)
  with pytest.raises(TypeError, match='device trainer only'):
    deep.fit(x, ids, t5)
  with pytest.raises(TypeError, match='device trainer only'):
    deep.fit_concatenated(x[0], ids[0], t5)
  with pytest.raises(TypeError, match='device trainer only'):
    deep.fit(x[0], ids[0], t5)
