"""The UIS-RNN model class with the public surface of `/root/reference/uisrnn/uisrnn.py`
(`UISRNN(args)`, `.fit`, `.fit_concatenated`, `.predict`, `.predict_single`, `.save`, `.load`,
`parallel_predict`, and the module-level `CoreRNN` / `BeamState`).

Inference on a CUDA device runs the whole beam search inside libuisrnn_b200.so (hand-written
sm_90a kernels behind the C ABI in include/uisrnn_b200.h): `predict(list)` hands all utterances
to ONE native call, which shards them over persistent CTAs; nothing but the labels comes back.
There is no silent fallback: on a CUDA device an unsupported configuration raises.  On the CPU
device (explicit `--enable_cuda=False`, the reference's own device rule) the decoder in
`beam_cpu.py` is used.  Training uses PyTorch autograd on the model's device.
"""
import collections
import functools
import threading
import warnings

import numpy as np
import torch
from torch import multiprocessing
from torch import nn
from torch import optim
import torch.nn.functional as F

from . import beam_cpu
from . import logger as logger_lib
from . import loss_func
from . import utils

_INITIAL_SIGMA2_VALUE = 0.1
# One utterance's N-best result (predict(..., n_best=k)): up to k hypotheses in rank order -- their label lists (the
# last tiled copy), their neg_likelihood over the whole decode and their cluster counts.
NBest = collections.namedtuple('NBest', ['labels', 'scores', 'speakers'])
# One utterance's score(..., per_frame=True): the neg_likelihood of the labelling and its per-frame increments (float32
# ndarray [N]; summed in fp32 in frame order they give `total` bit for bit).
FrameScores = collections.namedtuple('FrameScores', ['total', 'increments'])

_DEFAULT_KCAP = 0  # clusters per hypothesis held in device tables: 0 = the library's default (16 or 32, by kernel); grown on overflow


class CoreRNN(nn.Module):
  """GRU (+ dropout between layers when depth >= 2) followed by a two-layer MLP that predicts
  the mean of the next observation (uisrnn.py:32-52 of the reference; same parameter names, so
  `state_dict()`s are interchangeable)."""

  def __init__(self, input_dim, hidden_size, depth, observation_dim, dropout=0):
    super().__init__()
    self.hidden_size = hidden_size
    gru_kwargs = {'dropout': dropout} if depth >= 2 else {}
    self.gru = nn.GRU(input_dim, hidden_size, depth, **gru_kwargs)
    self.linear_mean1 = nn.Linear(hidden_size, hidden_size)
    self.linear_mean2 = nn.Linear(hidden_size, observation_dim)

  def forward(self, input_seq, hidden=None):
    output_seq, hidden = self.gru(input_seq, hidden)
    if isinstance(output_seq, nn.utils.rnn.PackedSequence):
      output_seq, _ = nn.utils.rnn.pad_packed_sequence(output_seq, batch_first=False)
    return self.linear_mean2(F.relu(self.linear_mean1(output_seq))), hidden


class BeamState:
  """Plain record of one beam-search hypothesis (uisrnn.py:55-77).  Kept for API compatibility;
  the CUDA path keeps the equivalent state on the device (slot pool + per-hypothesis tables)."""

  def __init__(self, source=None):
    if not source:
      self.mean_set, self.hidden_set, self.trace, self.block_counts = [], [], [], []
      self.neg_likelihood = 0
    else:
      self.mean_set = source.mean_set.copy()
      self.hidden_set = source.hidden_set.copy()
      self.trace = source.trace.copy()
      self.block_counts = source.block_counts.copy()
      self.neg_likelihood = source.neg_likelihood

  def append(self, mean, hidden, cluster):
    self.mean_set.append(mean.clone())
    self.hidden_set.append(hidden.clone())
    self.block_counts.append(1)
    self.trace.append(cluster)


def _check_test_sequence(test_sequence, observation_dim):
  """Input validation of predict_single (uisrnn.py:511-521): same exceptions, same order."""
  if not isinstance(test_sequence, np.ndarray) or test_sequence.dtype != float:
    raise TypeError('test_sequence should be a numpy array of float type.')
  if test_sequence.ndim != 2:
    raise ValueError('test_sequence must be 2-dim array.')
  if test_sequence.shape[1] != observation_dim:
    raise ValueError('test_sequence does not match the dimension specified by args.observation_dim.')


_TENSOR_DTYPES = (torch.float32, torch.float16, torch.bfloat16, torch.float64)


def _tensor_sequences(sequences, observation_dim, device, name='test_sequence'):
  """Whether a list of sequences holds torch tensors (True) or not (False: the ndarray rules apply).  Tensors are
  checked here: one dtype for the whole call, one of _TENSOR_DTYPES (TypeError), 2-D [N, observation_dim] (the
  ValueErrors of _check_test_sequence) and on `device` (ValueError).  A list mixing tensors with anything else is a
  TypeError.  `name` is the argument the messages name (test_sequence or train_sequence)."""
  is_tensor = [isinstance(s, torch.Tensor) for s in sequences]
  if not any(is_tensor):
    return False
  if not all(is_tensor):
    raise TypeError('{}s must be all numpy arrays or all torch tensors, not a mix of both.'.format(name))
  dtypes = sorted({str(s.dtype) for s in sequences})
  if len(dtypes) > 1:
    raise TypeError('all {} tensors of one call must share a dtype, got {}.'.format(name, ', '.join(dtypes)))
  if sequences[0].dtype not in _TENSOR_DTYPES:
    raise TypeError('{} tensors must be float32, float16, bfloat16 or float64, got {}.'.format(
        name, sequences[0].dtype))
  for sequence in sequences:
    if sequence.ndim != 2:
      raise ValueError('{} must be 2-dim array.'.format(name))
    if sequence.shape[1] != observation_dim:
      raise ValueError('{} does not match the dimension specified by args.observation_dim.'.format(name))
    if sequence.device != device:
      raise ValueError('{} tensors must be on the model\'s device {}, got {}.'.format(name, device, sequence.device))
  return True


def _fit_labels(train_cluster_ids, lengths, device):
  """The label sequences of a fit from tensors, on the host: every integer tensor [N] on `device` (any integer dtype and
  strides) becomes the list of str(v) of its values v (utils.host_labels, one read-back for all of them); host label
  sequences are kept for utils.concatenate_training_data to check.  A label tensor of another dtype is a TypeError, of
  another shape, length or device a ValueError."""
  if not isinstance(train_cluster_ids, list):
    return train_cluster_ids  # (concatenate_training_data raises the reference's TypeError)
  for u, ids in enumerate(train_cluster_ids):
    if isinstance(ids, torch.Tensor) and ids.device != device:
      raise ValueError('utterance {}: the label tensor is on {}, the sequences on {}'.format(u, ids.device, device))
  labels = utils.host_labels(train_cluster_ids)  # (dtype and shape checks)
  for u, (ids, n) in enumerate(zip(train_cluster_ids, lengths)):
    if isinstance(ids, torch.Tensor) and ids.shape[0] != n:
      raise ValueError('utterance {}: {} labels for {} frames'.format(u, ids.shape[0], n))
  return labels


def _device_rows(tensors):
  """(x, offsets) of checked tensors: one contiguous fp32 [rows, D] CUDA tensor (the caller's own when a single
  contiguous fp32 tensor starting on a 16-byte boundary is given, else one cat + cast, float64 rounded to nearest) and
  int64 frame offsets [U + 1].  The input projection reads the rows with float4 loads, so a view at an element offset
  that is not a multiple of 4 is copied."""
  offsets = np.zeros(len(tensors) + 1, np.int64)
  np.cumsum([t.shape[0] for t in tensors], out=offsets[1:])
  with torch.no_grad():
    t0 = tensors[0] if len(tensors) == 1 else None
    if t0 is not None and t0.dtype == torch.float32 and t0.is_contiguous() and t0.data_ptr() % 16 == 0:
      x = t0.detach()
    else:
      x = torch.cat([t.detach() for t in tensors]).to(torch.float32).contiguous()
  return x, offsets


def _device_ids(test_cluster_ids, lengths, device):
  """One contiguous int64 CUDA tensor [rows] of the label sequences of a tensor score() call: an integer tensor on
  `device` is taken with its values as they are (any strides: a strided one is copied), a host sequence is renamed on
  the host (canonical_labels: any hashable values) and uploaded."""
  parts = []
  for u, (ids, n) in enumerate(zip(test_cluster_ids, lengths)):
    if isinstance(ids, torch.Tensor):
      if ids.dtype.is_floating_point or ids.dtype.is_complex or ids.dtype == torch.bool:
        raise TypeError('utterance {}: a label tensor must have an integer dtype, got {}'.format(u, ids.dtype))
      if ids.device != device:
        raise ValueError('utterance {}: the label tensor is on {}, the sequences on {}'.format(u, ids.device, device))
      if ids.ndim != 1:
        raise ValueError('a label sequence must be a 1-D sequence of labels')
      part = ids.detach().to(torch.int64).contiguous()  # (an int64 tensor comes back as itself, strides included)
    else:
      part = torch.from_numpy(canonical_labels(ids).astype(np.int64)).to(device, non_blocking=True)
    if part.shape[0] != n:
      raise ValueError('utterance {}: {} labels for {} frames'.format(u, part.shape[0], n))
    parts.append(part)
  return torch.cat(parts) if len(parts) > 1 else parts[0]


class _Fingerprint:
  """Parameter tensors (copied, or the live ones) and scalars, compared exactly: per device, one fused difference and
  one fused max-norm of the tensors there, and one device -> host copy."""

  def __init__(self, tensors, scalars, copy):
    with torch.no_grad():
      self.tensors = [t.detach().clone() if copy else t.detach() for t in tensors]
    self.scalars = scalars

  def __eq__(self, other):
    if not isinstance(other, _Fingerprint) or self.scalars != other.scalars or len(self.tensors) != len(other.tensors):
      return False
    by_device = {}  # the parameters need not share a device (callers assign rnn_init_hidden / sigma2 freely)
    for a, b in zip(self.tensors, other.tensors):
      if a.shape != b.shape or a.dtype != b.dtype or a.device != b.device:
        return False
      by_device.setdefault(a.device, []).append((a, b))
    with torch.no_grad():
      for pairs in by_device.values():
        diff = torch._foreach_sub([a for a, _ in pairs], [b for _, b in pairs])  # pylint: disable=protected-access
        worst = torch.stack(torch._foreach_norm(diff, float('inf'))).max()  # pylint: disable=protected-access
        if not worst.item() == 0:  # NaN (a NaN element, or inf - inf) is unequal
          return False
    return True

  __hash__ = None


class UISRNN:
  """Unbounded Interleaved-State Recurrent Neural Network."""

  def __init__(self, args):
    self.observation_dim = args.observation_dim
    # uisrnn.py:97-98 pins 'cuda:0'; here it is the process's CURRENT device (0 unless the caller ran
    # torch.cuda.set_device, as one-process-per-GPU launches do)
    if torch.cuda.is_available() and args.enable_cuda:
      self.device = torch.device('cuda', torch.cuda.current_device())
    else:
      self.device = torch.device('cpu')
    self.rnn_model = CoreRNN(self.observation_dim, args.rnn_hidden_size, args.rnn_depth,
                             self.observation_dim, args.rnn_dropout).to(self.device)
    self.rnn_init_hidden = nn.Parameter(torch.zeros(args.rnn_depth, 1, args.rnn_hidden_size).to(self.device))
    self.estimate_sigma2 = (args.sigma2 is None)
    self.estimate_transition_bias = (args.transition_bias is None)
    sigma2 = _INITIAL_SIGMA2_VALUE if self.estimate_sigma2 else args.sigma2
    self.sigma2 = nn.Parameter(sigma2 * torch.ones(self.observation_dim).to(self.device))
    self.transition_bias = args.transition_bias
    self.transition_bias_denominator = 0.0
    self.crp_alpha = args.crp_alpha
    self.logger = logger_lib.Logger(args.verbosity)
    self._native = None          # (fingerprint, NativeModel) cache for the CUDA decoder
    self._native_lock = threading.Lock()
    if self.device.type == 'cuda':
      # say so NOW if the sm_90a kernels cannot hold this model (predict() / fit() would raise NativeError later;
      # there is no silent fallback): hidden <= 1024, dim <= 512, 1..4 GRU layers at every such size
      too_big = args.rnn_hidden_size > 1024 or self.observation_dim > 512 or args.rnn_depth > 4
      if too_big:
        self.logger.print(
            1, 'Warning: the CUDA kernels of this build hold models up to rnn_hidden_size=1024, observation_dim=512, '
               'rnn_depth=4; predict() on this device will raise for this model. Use --enable_cuda=False for it.')

  def __getstate__(self):
    # the device-side twin and its lock are per-process; pickled copies (forkserver workers of
    # parallel_predict) rebuild them on demand
    state = dict(self.__dict__)
    state['_native'] = None
    state['_native_lock'] = None
    return state

  def __setstate__(self, state):
    self.__dict__.update(state)
    self._native_lock = threading.Lock()

  # ------------------------------------------------------------------ persistence
  def save(self, filepath):
    """Writes the checkpoint dictionary of the reference (uisrnn.py:135-147), so files are
    interchangeable between the two implementations."""
    torch.save({
        'rnn_state_dict': self.rnn_model.state_dict(),
        'rnn_init_hidden': self.rnn_init_hidden.detach().cpu().numpy(),
        'transition_bias': self.transition_bias,
        'transition_bias_denominator': self.transition_bias_denominator,
        'crp_alpha': self.crp_alpha,
        'sigma2': self.sigma2.detach().cpu().numpy()}, filepath)

  def load(self, filepath):
    """Restores a checkpoint written by `save` (of this package or of the reference).  The file
    holds numpy arrays, so it is read with `weights_only=False` (the reference's plain
    `torch.load`, uisrnn.py:155, fails on torch >= 2.6)."""
    var_dict = torch.load(filepath, map_location=self.device, weights_only=False)
    self.rnn_model.load_state_dict(var_dict['rnn_state_dict'])
    self.rnn_init_hidden = nn.Parameter(torch.from_numpy(var_dict['rnn_init_hidden']).to(self.device))
    self.transition_bias = float(var_dict['transition_bias'])
    self.transition_bias_denominator = float(var_dict['transition_bias_denominator'])
    self.crp_alpha = float(var_dict['crp_alpha'])
    self.sigma2 = nn.Parameter(torch.from_numpy(var_dict['sigma2']).to(self.device))
    self._native = None
    self.logger.print(
        3, 'Loaded model with transition_bias={}, crp_alpha={}, sigma2={}, rnn_init_hidden={}'.format(
            self.transition_bias, self.crp_alpha, var_dict['sigma2'], var_dict['rnn_init_hidden']))

  # ------------------------------------------------------------------ training
  def _get_optimizer(self, optimizer, learning_rate):
    groups = [{'params': self.rnn_model.parameters()}, {'params': self.rnn_init_hidden}]
    if self.estimate_sigma2:
      groups.append({'params': self.sigma2})
    assert optimizer == 'adam', 'Only adam optimizer is supported.'
    return optim.Adam(groups, lr=learning_rate)

  def fit_concatenated(self, train_sequence, train_cluster_id, args):
    """Trains on one concatenated sequence `train_sequence` [N, D] (float64) with string labels
    `train_cluster_id` [N] (uisrnn.py:172-313): per iteration a random batch of per-speaker
    sub-sequences, running-mean prediction, weighted-MSE + sigma^2 prior + norm regulariser,
    clipped Adam step, sigma^2 >= 1e-6.

    A CUDA model also takes a torch tensor [N, D] on its device with an integer label tensor [N] or host labels: see
    `fit`."""
    if self.device.type == 'cuda' and isinstance(train_sequence, torch.Tensor):
      _tensor_sequences([train_sequence], self.observation_dim, self.device, 'train_sequence')
      self._require_device_trainer(args)
      train_cluster_id = _fit_labels([train_cluster_id], [train_sequence.shape[0]], self.device)[0]
      if isinstance(train_cluster_id, list):
        train_cluster_id = np.array(train_cluster_id)
      if (not isinstance(train_cluster_id, np.ndarray) or
          not train_cluster_id.dtype.name.startswith(('str', 'unicode'))):
        raise TypeError('train_cluster_id type be a numpy array of strings.')
      if train_cluster_id.ndim != 1:
        raise ValueError('train_cluster_id must be 1-dim array.')
      if train_sequence.shape[0] != len(train_cluster_id):
        raise ValueError('train_sequence length is not equal to train_cluster_id length.')
      self._fit_tensors([train_sequence], train_cluster_id, args)
      return
    if not isinstance(train_sequence, np.ndarray) or train_sequence.dtype != float:
      raise TypeError('train_sequence should be a numpy array of float type.')
    if isinstance(train_cluster_id, list):
      train_cluster_id = np.array(train_cluster_id)
    if (not isinstance(train_cluster_id, np.ndarray) or
        not train_cluster_id.dtype.name.startswith(('str', 'unicode'))):
      raise TypeError('train_cluster_id type be a numpy array of strings.')
    if train_sequence.ndim != 2:
      raise ValueError('train_sequence must be 2-dim array.')
    if train_cluster_id.ndim != 1:
      raise ValueError('train_cluster_id must be 1-dim array.')
    total_length, observation_dim = train_sequence.shape
    if observation_dim != self.observation_dim:
      raise ValueError('train_sequence does not match the dimension specified by args.observation_dim.')
    if total_length != len(train_cluster_id):
      raise ValueError('train_sequence length is not equal to train_cluster_id length.')

    self.rnn_model.train()
    optimizer = self._get_optimizer(optimizer=args.optimizer, learning_rate=args.learning_rate)
    if self._native_fit_supported(args):
      self._sync_replicas()
    if self._native_fit_supported(args):
      # device-resident training set: row indices per sub-sequence instead of num_permutations copies
      index_lists, seq_lengths = utils.resize_indices(train_cluster_id, args.num_permutations)
      self._fit_native(train_sequence, index_lists, seq_lengths, args)
      return
    self.last_fit_backend = 'torch'
    sub_sequences, seq_lengths = utils.resize_sequence(
        sequence=train_sequence, cluster_id=train_cluster_id, num_permutations=args.num_permutations)
    batch = None
    if args.batch_size is None:  # "batch learning": one fixed batch holding every sub-sequence
      batch = utils.pack_sequence(sub_sequences, seq_lengths, None, self.observation_dim, self.device)
    for num_iter in range(args.train_iteration):
      optimizer.zero_grad()
      if args.batch_size is not None:
        batch = utils.pack_sequence(sub_sequences, seq_lengths, args.batch_size, self.observation_dim,
                                    self.device)
      packed_input, rnn_truth = batch
      width = rnn_truth.size(1)
      mean, _ = self.rnn_model(packed_input, self.rnn_init_hidden.repeat(1, width, 1))
      # running average of the predictions over time (uisrnn.py:265-271 does it with a dense
      # diag(1/t) matrix product; the values are identical)
      steps = torch.arange(1, mean.size(0) + 1, device=self.device).float()
      mean = torch.cumsum(mean, dim=0) * (1.0 / steps).view(-1, 1, 1)
      mask = (rnn_truth != 0).float()
      weight = 1 / (2 * self.sigma2)
      loss1 = loss_func.weighted_mse_loss(input_tensor=mask * mean[:-1, :, :], target_tensor=rnn_truth,
                                          weight=weight)
      residual2 = ((mask * mean[:-1, :, :] - rnn_truth) ** 2).view(-1, observation_dim)
      num_non_zero = torch.sum((residual2 != 0).float(), dim=0).squeeze()
      loss2 = loss_func.sigma2_prior_loss(num_non_zero, args.sigma_alpha, args.sigma_beta, self.sigma2)
      loss3 = loss_func.regularization_loss(self.rnn_model.parameters(), args.regularization_weight)
      loss = loss1 + loss2 + loss3
      loss.backward()
      nn.utils.clip_grad_norm_(self.rnn_model.parameters(), args.grad_max_norm)
      optimizer.step()
      self.sigma2.data.clamp_(min=1e-6)
      if num_iter % 10 == 0 or num_iter == args.train_iteration - 1:
        self.logger.print(
            2, 'Iter: {:d}  \tTraining Loss: {:.4f}    \n    Negative Log Likelihood: {:.4f}\t'
               'Sigma2 Prior: {:.4f}\tRegularization: {:.4f}'.format(
                   num_iter, float(loss.data), float(loss1.data), float(loss2.data), float(loss3.data)))
    self._native = None
    self.logger.print(1, 'Done training with {} iterations'.format(args.train_iteration))

  def _sync_replicas(self):
    """Data-parallel fit(): inside an initialised `torch.distributed` job every rank adopts rank 0's
    parameters and host RNG state (numpy + `random`), so the shuffle of `concatenate_training_data`, the
    permutations of `resize_sequence` and every mini-batch draw are the same on all ranks.  No-op in a
    single process."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
      return
    with torch.no_grad():
      for tensor in list(self.rnn_model.state_dict().values()) + [self.rnn_init_hidden.data, self.sigma2.data]:
        dist.broadcast(tensor, src=0)
    import random
    rng = [np.random.get_state(), random.getstate()]  # utils.py draws from both generators
    dist.broadcast_object_list(rng, src=0)
    np.random.set_state(rng[0])
    random.setstate(rng[1])

  def _native_fit_supported(self, args):
    """On a CUDA device fit() runs on the hand-written training kernels (csrc/uis_train.cu): 1..4 stacked GRU
    layers (inter-layer dropout in train mode), any mini-batch width including batch_size=None (one batch of
    every sub-sequence).  The CPU device always trains with PyTorch, as the reference does."""
    del args
    return self.device.type == 'cuda' and 1 <= self.rnn_init_hidden.shape[0] <= 4

  def _require_device_trainer(self, args):
    if not self._native_fit_supported(args):
      raise TypeError('train_sequence tensors train on the device trainer only (rnn_depth 1 to 4 on a CUDA device); '
                      'this model trains with PyTorch: pass float64 numpy arrays.')

  def _fit_tensors(self, sequences, train_cluster_id, args):
    """fit_concatenated of checked CUDA tensors `sequences`, whose rows back to back are the concatenated sequence, and
    their string labels: the steps of the ndarray path on the device trainer, reading the rows in place."""
    self.rnn_model.train()
    self._get_optimizer(optimizer=args.optimizer, learning_rate=args.learning_rate)
    self._sync_replicas()
    index_lists, seq_lengths = utils.resize_indices(train_cluster_id, args.num_permutations)
    self._fit_native(sequences, index_lists, seq_lengths, args)

  def _fit_native(self, train_sequence, index_lists, seq_lengths, args):
    """fit_concatenated's iteration loop (uisrnn.py:252-311) on libuisrnn_b200.so: the training set,
    parameters, gradients and Adam state stay on the device; per iteration only the ids of the drawn
    sub-sequences go up (the batch is gathered on the device) and the loss scalars are read back
    when they are logged.  `train_sequence` is a float64 ndarray (copied to the device as fp32, steps on stream 0) or a
    list of CUDA tensors (read in place; every step on torch's current stream of the model's device)."""
    from . import native
    import torch.distributed as dist
    world = dist.get_world_size() if (dist.is_available() and dist.is_initialized()) else 1
    rank = dist.get_rank() if world > 1 else 0
    # world > 1: data-parallel fit (SURVEY 8(e), optional) -- every rank holds rank 0's parameters and draws
    # the SAME mini-batches (_sync_replicas); rank r owns batch columns r, r + world, ...
    state = {k: v.detach().cpu().numpy() for k, v in self.rnn_model.state_dict().items()}
    depth = int(self.rnn_init_hidden.shape[0])
    order = native.param_order(depth)
    params = {name: state[name] for name in order[:-2]}
    params['rnn_init_hidden'] = self.rnn_init_hidden.detach().cpu().numpy().reshape(-1)
    params['sigma2'] = self.sigma2.detach().cpu().numpy()
    # the dropout masks of the stacked GRU are seeded from torch's generator (so torch.manual_seed() makes a run
    # repeatable, as it does for the reference), one draw per fit_concatenated call (in a data-parallel job every
    # rank masks its own columns, so the ranks need not share the seed)
    dropout = float(self.rnn_model.gru.dropout) if depth > 1 else 0.0
    dropout_seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if dropout > 0 else 0
    hparams = {'learning_rate': args.learning_rate, 'sigma_alpha': args.sigma_alpha, 'sigma_beta': args.sigma_beta,
               'regularization_weight': args.regularization_weight, 'grad_max_norm': args.grad_max_norm,
               'train_sigma2': self.estimate_sigma2, 'rnn_depth': depth, 'rnn_dropout': dropout,
               'dropout_seed': dropout_seed}
    trainer = native.NativeTrainer(params, hparams, device=self.device.index or 0)
    self.last_training_losses = []
    self.last_training_loss_terms = []  # [iteration] -> (negative log likelihood, sigma2 prior, regularisation)
    self.last_fit_backend = 'native'
    comm = torch.zeros(trainer.comm_size(), dtype=torch.float32, device=self.device) if world > 1 else None
    sampler = utils.BatchSampler(seq_lengths, args.batch_size)
    tensors = isinstance(train_sequence, list)
    stream = torch.cuda.current_stream(self.device).cuda_stream if tensors else 0
    try:
      if tensors:
        trainer.set_corpus_device(train_sequence, index_lists, stream=stream)
      else:
        trainer.set_corpus(train_sequence, index_lists)
      pending = 0  # steps enqueued since the losses were last read back
      for num_iter in range(args.train_iteration):
        chosen, _ = sampler.draw()  # same np.random.choice call as utils.pack_sequence
        if world == 1:
          trainer.step_corpus(chosen, stream=stream)  # asynchronous: the host runs ahead of the device
        else:
          # local forward/backward on this rank's columns -> ONE all-reduce(sum) of [gradients | loss
          # statistics] over NCCL -> identical normalise / clip / Adam step on every rank
          mine = shard_columns(len(chosen), rank, world)
          if len(mine):
            trainer.step_corpus(chosen[mine], mode=2, stream=stream)
            trainer.comm_export(comm.data_ptr(), stream=stream)
          else:
            comm.zero_()
          dist.all_reduce(comm, op=dist.ReduceOp.SUM)
          trainer.comm_apply(comm.data_ptr(), stream=stream)
        pending += 1
        log_now = num_iter % 10 == 0 or num_iter == args.train_iteration - 1
        if log_now or pending == 4096:
          recent = trainer.losses(pending)
          self.last_training_losses.extend(float(v) for v in recent[:, 0])
          self.last_training_loss_terms.extend(tuple(float(v) for v in row) for row in recent)
          pending = 0
          if log_now:
            loss1, loss2, loss3 = (float(v) for v in recent[-1])
            self.logger.print(
                2, 'Iter: {:d}  \tTraining Loss: {:.4f}    \n    Negative Log Likelihood: {:.4f}\t'
                   'Sigma2 Prior: {:.4f}\tRegularization: {:.4f}'.format(
                       num_iter, loss1 + loss2 + loss3, loss1, loss2, loss3))
      trained = trainer.parameters()
    finally:
      trainer.close()
    with torch.no_grad():
      self.rnn_model.load_state_dict({k: torch.from_numpy(trained[k].copy()) for k in order[:-2]})
      self.rnn_init_hidden.data.copy_(torch.from_numpy(trained['rnn_init_hidden'].reshape(depth, 1, -1)))
      self.sigma2.data.copy_(torch.from_numpy(trained['sigma2']))
    self._native = None
    self.logger.print(1, 'Done training with {} iterations'.format(args.train_iteration))

  def fit(self, train_sequences, train_cluster_ids, args):
    """Trains on a list of sequences (+ list of label sequences) or on one concatenated sequence
    (uisrnn.py:315-386).  Estimates / running-averages `transition_bias` unless it was given.

    Training sets already on the GPU (not in the reference): a CUDA model that trains on the device trainer (rnn_depth
    1 to 4) also takes a list of torch tensors [N_i, D], or one tensor as the concatenated form, on the model's device,
    all float32, all float16, all bfloat16 or all float64 (any strides; requires_grad is ignored).  A list mixing
    tensors with ndarrays, or mixing dtypes, is a TypeError.  A label sequence may then be an integer tensor [N_i] on
    the same device (any integer dtype and strides) or host labels as above, in any mix per utterance; an integer
    label v is the string str(v), so it trains exactly as that string would, uniqueness prefixes included.  The label
    tensors are read back to the host once: the shuffle, the sub-sequence permutations and the mini-batch draws stay
    on the host and use the same random numbers as for ndarrays.  The trainer reads the rows in place, in their dtype,
    on torch's current stream of the device, with no copy of the training set (a tensor whose elements are not in
    unit stride is copied once).  With the same seeds every iteration gathers, bit for bit, the batch a fit of the same
    values as float64 ndarrays gathers (float64 rounds to nearest on the device as the ndarray path's cast does, float16
    / bfloat16 convert exactly), so a step's gradients are those of the ndarray route.  Whole fits agree as two ndarray
    fits do: to the trainer's run-to-run spread (its per-dimension residual sums are float atomics).  The rows must not
    change until fit() returns.  A CPU model raises the reference's TypeError
    for tensors, and a CUDA model that trains with PyTorch (rnn_depth > 4) a TypeError."""
    on_cuda = self.device.type == 'cuda'
    if not on_cuda and isinstance(train_sequences, list) and any(isinstance(s, torch.Tensor) for s in train_sequences):
      raise TypeError('train_sequence should be a numpy array of float type.')
    if isinstance(train_sequences, np.ndarray) or (on_cuda and isinstance(train_sequences, torch.Tensor)):
      if self.estimate_transition_bias:
        self.logger.print(
            2, 'Warning: transition_bias cannot be correctly estimated from a concatenated sequence; '
               'train_sequences will be treated as a single sequence. This can lead to inaccurate '
               'estimation of transition_bias. Please, consider estimating transition_bias before '
               'concatenating the sequences and passing it as argument.')
      train_sequences = [train_sequences]
      train_cluster_ids = [train_cluster_ids]
    elif not isinstance(train_sequences, list):
      raise TypeError('train_sequences must be a list or numpy.ndarray')
    tensors = on_cuda and _tensor_sequences(train_sequences, self.observation_dim, self.device, 'train_sequence')
    if tensors:
      self._require_device_trainer(args)
      train_cluster_ids = _fit_labels(train_cluster_ids, [s.shape[0] for s in train_sequences], self.device)
    if self._native_fit_supported(args):
      self._sync_replicas()  # before the shuffle inside concatenate_training_data
    if self.estimate_transition_bias:
      bias, denominator = utils.estimate_transition_bias(train_cluster_ids)
      if self.transition_bias is None:
        self.transition_bias = bias
        self.transition_bias_denominator = denominator
      else:  # weighted running average over successive fit() calls
        merged = self.transition_bias_denominator + denominator
        self.transition_bias = (self.transition_bias * self.transition_bias_denominator +
                                bias * denominator) / merged
        self.transition_bias_denominator = merged
    sequence, cluster_id = utils.concatenate_training_data(
        train_sequences, train_cluster_ids, args.enforce_cluster_id_uniqueness, True)
    if tensors:
      self._fit_tensors(sequence, cluster_id, args)
    else:
      self.fit_concatenated(sequence, cluster_id, args)

  # ------------------------------------------------------------------ inference
  def _fingerprint(self, copy=True):
    """Identity of the parameter values the device-side twin is built from: equal to another fingerprint exactly when
    every parameter has the same shape, dtype, device and elements (a NaN never equals), and the decoding scalars are
    equal.  `_version` does not move on edits through `.data` (an idiom the reference's own tests use), and norms
    miss edits that keep every |value| (a sign flip, a swap of rows), so the twin keeps a copy of the parameters
    (copy=True) and each call compares the live ones (copy=False) with it."""
    tensors = list(self.rnn_model.parameters()) + [self.rnn_init_hidden, self.sigma2]
    return _Fingerprint(tensors, (self.transition_bias, self.crp_alpha), copy)

  def export_weights(self):
    """Weights as float32 numpy arrays in the layout libuisrnn_b200.so / the oracle expect."""
    state = {k: v.detach().cpu().numpy() for k, v in self.rnn_model.state_dict().items()}
    depth = self.rnn_init_hidden.shape[0]
    out = {'depth': depth,
           'w1': state['linear_mean1.weight'], 'b1': state['linear_mean1.bias'],
           'w2': state['linear_mean2.weight'], 'b2': state['linear_mean2.bias'],
           'h0': self.rnn_init_hidden.detach().cpu().numpy(),
           'sigma2': self.sigma2.detach().cpu().numpy(),
           'transition_bias': self.transition_bias, 'crp_alpha': self.crp_alpha}
    for layer in range(depth):
      for name in ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh'):
        out['{}_l{}'.format(name, layer)] = state['gru.{}_l{}'.format(name, layer)]
    return out

  def _native_model(self, device_index=None):
    """The device-side twin of this model (created lazily, rebuilt when any parameter changed)."""
    from . import native  # raises NativeError if the library has not been built
    index = (self.device.index or 0) if device_index is None else device_index
    with self._native_lock:
      if self._native is None or self._native[0] != (self._fingerprint(copy=False), index):
        if self.transition_bias is None:
          raise TypeError('transition_bias is not set: call fit() or pass --transition_bias.')
        self._native = ((self._fingerprint(), index), native.NativeModel(self.export_weights(), device=index))
      return self._native[1]

  def _decode(self, sequences, args, bounds, n_best, pairs, as_arrays=False, tensors=False):
    """The one decode behind every predict entry point, of checked `sequences` under speaker `bounds` ((max, min) int32
    arrays from native.speaker_bounds, None = absent), `n_best` and `pairs` (checked (crp_alpha, transition_bias) pairs,
    None = the model's own).  Returns (hypotheses, speakers): hypotheses[c][u] is the NBest of utterance u under pair c
    with n_best, else its hypothesis 0's labels (an int32 array on CUDA with as_arrays, else a list of ints; empty for
    an empty utterance); speakers[c][u] is the cluster count of hypothesis 0 (0 for an empty utterance).  With
    `tensors` the sequences are CUDA tensors and so are the labels, scores and cluster counts of the hypotheses."""
    if tensors:
      return _native_decode_tensors(self._native_model(), sequences, args, bounds, n_best, pairs)
    if self.device.type == 'cuda':
      return _native_decode(self._native_model(), sequences, args, bounds, n_best, pairs, as_arrays)
    mx, mn = bounds
    hyps, speakers = [], []
    for alpha, bias in pairs or [(self.crp_alpha, self.transition_bias)]:
      decoder = beam_cpu.CpuBeamSearch(self, crp_alpha=alpha, transition_bias=bias)
      outs = [decoder.decode(s, args.beam_size, args.look_ahead, args.test_iteration,
                             int(mx[u]) if mx is not None else 0, int(mn[u]) if mn is not None else 0,
                             n_best=n_best or 1) for u, s in enumerate(sequences)]
      hyps.append([NBest(*o) if n_best else (o[0][0] if o[0] else []) for o in outs])
      speakers.append([o[2][0] if o[2] else 0 for o in outs])
    return hyps, speakers

  def _predict(self, test_sequences, args, max_speakers, min_speakers, n_best, pairs):
    """predict() of an ndarray or a list, after decode_params was checked (pairs, None = none given)."""
    on_cuda = self.device.type == 'cuda'
    single = isinstance(test_sequences, np.ndarray) or (on_cuda and isinstance(test_sequences, torch.Tensor))
    if not single and not isinstance(test_sequences, list):
      raise TypeError('test_sequences should be either a list or numpy array.')
    sequences = [test_sequences] if single else test_sequences
    tensors = on_cuda and _tensor_sequences(sequences, self.observation_dim, self.device)
    if not tensors:
      for sequence in sequences:
        _check_test_sequence(sequence, self.observation_dim)
    if single and (np.ndim(max_speakers) or np.ndim(min_speakers)):
      raise ValueError('predict_single takes one int per bound')
    k = _check_n_best(n_best, args) if n_best is not None else None
    bounds = _speaker_bounds(len(sequences), max_speakers, min_speakers)
    hyps, speakers = self._decode(sequences, args, bounds, k, pairs, tensors=tensors)
    _warn_min_speakers([len(s) for s in sequences], speakers, bounds[1], pairs is not None, stacklevel=4)
    out = [row[0] for row in hyps] if single else hyps
    return out if pairs is not None else out[0]

  def predict_single(self, test_sequence, args, *, max_speakers=None, min_speakers=None, n_best=None):
    """Labels (list of N ints) for one test sequence [N, D] float64 (uisrnn.py:479-562).

    max_speakers / min_speakers (ints, 0 or None = no bound) bound the number of speakers, and n_best returns
    an NBest instead; a CUDA model also takes a torch tensor: see `predict`."""
    if not (self.device.type == 'cuda' and isinstance(test_sequence, torch.Tensor)):
      _check_test_sequence(test_sequence, self.observation_dim)
    return self._predict(test_sequence, args, max_speakers, min_speakers, n_best, None)

  def predict(self, test_sequences, args, *, max_speakers=None, min_speakers=None, n_best=None, decode_params=None):
    """Labels for one sequence (ndarray -> list of ints) or many (list -> list of lists)
    (uisrnn.py:564-590).  On CUDA a list is decoded by a single native call; a list whose workspace does not fit
    the free device memory is decoded inside that call in groups of whole utterances, one after the other, with the
    results of one group (UISRNN_B200_MAX_ROWS sets the frames per group).  This holds for tensors, n_best, bounds and
    decode_params too.

    Speaker bounds (not in the reference): `max_speakers` / `min_speakers` is an int for every utterance or one
    value per utterance, 0 or None = no bound.  A hypothesis never holds more than max_speakers clusters, so every
    label is < max_speakers.  The labels come from the best-ranked final hypothesis with at least min_speakers
    clusters; when the final beam holds none, rank 0's labels are returned and one warning names those utterances.
    Clusters are counted over the whole decode (test_iteration tiled copies), so with test_iteration > 1 the
    returned labels may use fewer distinct ids than min_speakers.

    N-best (not in the reference): with `n_best` = k (1 <= k <= beam_size) every utterance gives an `NBest`
    (labels, scores, speakers) instead of a label list: one NBest for an ndarray, a list of them for a list.  It holds
    up to k final hypotheses in rank order -- the first k final ranks with at least min_speakers clusters, or rank 0
    alone when none has them -- so hypothesis 0 is what the call returns without n_best.  `scores` are the
    hypotheses' neg_likelihood accumulated over the whole decode (lower is better; the gap between the first two is
    a confidence), `speakers` their cluster counts.  An empty sequence gives no hypothesis.  With test_iteration > 1
    two hypotheses can differ only in an earlier tiled copy and so carry the same labels; they are kept apart.

    Decoding-parameter sweeps (not in the reference): `decode_params` is a non-empty sequence of (crp_alpha,
    transition_bias) pairs, crp_alpha finite and > 0, transition_bias finite and in (0, 1).  The result is then a list
    with one entry per pair, entry c being exactly what this call returns without `decode_params` for a model whose
    crp_alpha / transition_bias are pair c (bounds and n_best apply to every pair).  The model is not changed.  On a
    CUDA device the whole grid is one native call: the inputs are copied and projected once.  Pick a pair by scoring
    each entry on a labelled dev set (e.g. `evals.compute_sequence_match_accuracy`).

    Inputs already on the GPU (not in the reference): a CUDA model also takes a torch tensor [N, D] or a list of them,
    on the model's device, all float32, all float16, all bfloat16 or all float64 (any strides; requires_grad is
    ignored).  A list mixing tensors with ndarrays, or mixing dtypes, is a TypeError.  The rows are cast to float32 on
    the device (float64 rounds to nearest as the ndarray path's cast does, so the same values decode bit for bit either
    way; float16 / bfloat16 decode as their exact float64 upcast would) and decoded on torch's current stream of the
    device, with nothing crossing the bus but the per-utterance counts the call reads back when it ends.  Every
    utterance then gives an int64 CUDA tensor [N] of labels instead of a list, and with n_best an NBest of CUDA tensors:
    labels int64 [n, N], scores float32 [n], speakers int32 [n], for the n hypotheses returned.  Bounds and
    decode_params behave as for ndarrays.  A CPU model raises the reference's TypeError for tensors."""
    pairs = _decode_params(decode_params) if decode_params is not None else None
    return self._predict(test_sequences, args, max_speakers, min_speakers, n_best, pairs)

  def score(self, test_sequences, test_cluster_ids, *, per_frame=False, decode_params=None):
    """The neg_likelihood the model gives to given speaker labellings (not in the reference, where it exists only
    inside the beam search): the score of the trace that assigns frame t to cluster test_cluster_ids[t], the same
    quantity as `NBest.scores` -- lower is better.  Scoring the ground truth against the decoded hypothesis tells a
    search error (the truth scores lower) from a model error.

    One sequence (float64 ndarray [N, D], validated as in `predict`) with one label sequence (N hashable values) gives
    a float; a list of sequences with a list of label sequences gives a list of floats.  Labels are taken up to
    renaming: they are mapped to 0, 1, 2, ... in order of first appearance.  test_iteration is not applied: the
    sequence is scored once, as given (tile both the sequence and its labels to score a tiled decode).  An empty
    sequence scores 0.  With per_frame=True every utterance gives a `FrameScores(total, increments)` instead.  On a
    CUDA device a list is scored by one native call, in groups of whole utterances when it does not fit the device at
    once (as `predict`; the scores are those of one group, bit for bit).

    With `decode_params` (a non-empty sequence of (crp_alpha, transition_bias) pairs, validated as in `predict`) the
    result is a list with one entry per pair, each being what this call returns for a model with that pair.  On a CUDA
    device the GRU work is done once for all pairs.

    Inputs already on the GPU: a CUDA model also takes torch tensors as `predict` does (same rules and casts).  Their
    label sequences may be integer CUDA tensors [N] on the same device (any integer dtype and any values, negative and
    beyond 32 bits included: they are renamed in order of first appearance on the device) or host label sequences as
    above.  A list of tensors then gives a float32 CUDA tensor [U] of scores, a single tensor a 0-d one, and
    decode_params a list of such tensors, one per pair; with per_frame every utterance gives a FrameScores of a 0-d total
    and float32 [N] increments.  The scores equal those of the ndarray call bit for bit.  The call enqueues its work on
    torch's current stream of the device and returns without waiting for it."""
    pairs = _decode_params(decode_params) if decode_params is not None else None
    if self.device.type == 'cuda' and isinstance(test_sequences, torch.Tensor):
      out = self.score([test_sequences], [test_cluster_ids], per_frame=per_frame, decode_params=pairs)
      return out[0] if pairs is None else [entry[0] for entry in out]
    if isinstance(test_sequences, np.ndarray):
      out = self.score([test_sequences], [test_cluster_ids], per_frame=per_frame, decode_params=pairs)
      return out[0] if pairs is None else [entry[0] for entry in out]
    if not isinstance(test_sequences, list):
      raise TypeError('test_sequences should be either a list or numpy array.')
    if not isinstance(test_cluster_ids, (list, tuple)):
      raise TypeError('test_cluster_ids should be a list with one label sequence per sequence.')
    if len(test_cluster_ids) != len(test_sequences):
      raise ValueError('{} sequences but {} label sequences'.format(len(test_sequences), len(test_cluster_ids)))
    if self.device.type == 'cuda' and _tensor_sequences(test_sequences, self.observation_dim, self.device):
      return self._score_tensors(test_sequences, test_cluster_ids, per_frame, pairs)
    for sequence in test_sequences:
      _check_test_sequence(sequence, self.observation_dim)
    labels = [canonical_labels(ids) for ids in test_cluster_ids]
    for u, (sequence, lab) in enumerate(zip(test_sequences, labels)):
      if len(lab) != len(sequence):
        raise ValueError('utterance {}: {} labels for {} frames'.format(u, len(lab), len(sequence)))
    if self.device.type == 'cuda':
      model = self._native_model()
      with model.lock:
        out = model.score_sweep(test_sequences, labels, pairs, per_frame=per_frame)
      totals, increments = out if per_frame else (out, None)
      result = [[FrameScores(float(v), inc[c]) for v, inc in zip(row, increments)] if per_frame else
                [float(v) for v in row] for c, row in enumerate(totals)]
    else:
      result = []
      for alpha, bias in pairs or [(self.crp_alpha, self.transition_bias)]:
        decoder = beam_cpu.CpuBeamSearch(self, crp_alpha=alpha, transition_bias=bias)
        out = [decoder.score(sequence, lab) for sequence, lab in zip(test_sequences, labels)]
        result.append([FrameScores(float(t), inc) for t, inc in out] if per_frame else [float(t) for t, _ in out])
    return result if pairs is not None else result[0]

  def _score_tensors(self, sequences, test_cluster_ids, per_frame, pairs):
    """score() of a list of checked CUDA tensors: one uis_score_device_ids call on torch's current stream, outputs
    allocated by torch on that stream, no synchronisation."""
    x, offsets = _device_rows(sequences)
    ids = _device_ids(test_cluster_ids, np.diff(offsets), self.device)
    n, rows, configs = len(sequences), int(offsets[-1]), 1 if pairs is None else len(pairs)
    scores = torch.empty((configs, n), dtype=torch.float32, device=self.device)
    frames = torch.empty((configs, rows), dtype=torch.float32, device=self.device) if per_frame else None
    model = self._native_model()
    with model.lock:
      model.score_device_ids(x.data_ptr(), offsets, ids.data_ptr(), scores.data_ptr(), pairs,
                             frame_ptr=frames.data_ptr() if per_frame else 0,
                             stream=torch.cuda.current_stream(self.device).cuda_stream)
    result = [[FrameScores(scores[c, u], frames[c, offsets[u]:offsets[u + 1]]) for u in range(n)] if per_frame else
              scores[c] for c in range(configs)]
    return result if pairs is not None else result[0]


def canonical_labels(ids):
  """int32 ndarray of a label sequence renamed to 0, 1, 2, ... in order of first appearance (any hashable values)."""
  if isinstance(ids, (str, bytes)) or np.ndim(ids) > 1:
    raise ValueError('a label sequence must be a 1-D sequence of labels')
  seen = {}
  return np.fromiter((seen.setdefault(v.item() if isinstance(v, np.generic) else v, len(seen)) for v in ids),
                     dtype=np.int32, count=len(ids))


def _speaker_bounds(n, max_speakers, min_speakers):
  from . import native  # validation only: the library is not loaded
  return native.speaker_bounds(n, max_speakers, min_speakers)


def _warn_min_speakers(lengths, speakers, min_speakers, swept, stacklevel, indices=None):
  """One warning naming the utterances (by `indices`, default their positions), or the (utterance, pair)s of a sweep,
  whose final beam held no hypothesis with min_speakers clusters.  speakers[c][u]: hypothesis 0's cluster count."""
  if min_speakers is None:
    return
  indices = range(len(lengths)) if indices is None else indices
  short = [(int(i), c) if swept else int(i) for c, row in enumerate(speakers)
           for i, n, k, lo in zip(indices, lengths, row, min_speakers) if n > 0 and k < lo]
  if short:
    warnings.warn('min_speakers: the final beam of {} {} held no hypothesis with that many speakers; the best '
                  'hypothesis was returned instead'.format('(utterance, pair)' if swept else 'utterance(s)', short),
                  RuntimeWarning, stacklevel=stacklevel)


def _decode_params(decode_params):
  """Validated list of (crp_alpha, transition_bias) float pairs (ValueError names the first bad pair)."""
  from . import native  # validation only: the library is not loaded
  alpha, bias = native.decode_params(decode_params)
  return [(float(a), float(b)) for a, b in zip(alpha, bias)]


def _check_n_best(n_best, args):
  from . import native  # validation only: the library is not loaded
  return native.check_n_best(n_best, args.beam_size)


def _native_decode(model, sequences, args, bounds, n_best, pairs, as_arrays=False):
  """UISRNN._decode on a NativeModel: one NativeModel.predict_sweep call, repeated with larger device tables (kcap)
  while a hypothesis opens more clusters than they hold (UIS_ERR_OVERFLOW)."""
  mx, mn = bounds
  labels, scores, speakers, count = _grow_kcap(model, lambda kcap: model.predict_sweep(
      sequences, pairs, beam_size=args.beam_size, look_ahead=args.look_ahead, test_iteration=args.test_iteration,
      kcap=kcap, max_speakers=mx, min_speakers=mn, n_best=n_best))
  if n_best is None:  # hypothesis 0's labels: label plane 0, which an empty utterance leaves empty
    hyps = [[lab[c, 0] if as_arrays else lab[c, 0].tolist() for lab in labels] for c in range(len(count))]
  else:
    hyps = [[NBest(lab[c, :n].tolist(), s[:n], k[:n]) for lab, s, k, n in zip(labels, sc, sp, cn)]
            for c, (sc, sp, cn) in enumerate(zip(scores.tolist(), speakers.tolist(), count.tolist()))]
  return hyps, speakers[:, :, 0]


def _grow_kcap(model, decode):
  """decode(kcap) under the model's lock, repeated with larger device tables (kcap) while a hypothesis opens more
  clusters than they hold (UIS_ERR_OVERFLOW)."""
  from . import native
  kcap = _DEFAULT_KCAP
  while True:
    try:
      with model.lock:  # a uis_model handle (one workspace) is not re-entrant
        return decode(kcap)
    except native.NativeError as err:
      if err.code != native.UIS_ERR_OVERFLOW or kcap >= 1024:
        raise
      kcap = 32 if kcap == 0 else kcap * 2


def _native_decode_tensors(model, tensors, args, bounds, n_best, pairs):
  """_native_decode of checked CUDA tensors: one uis_predict_device_sweep call on torch's current stream into outputs
  torch allocates there, then one synchronisation (NativeModel.stats raises what a job's status reports, e.g. the
  overflow that grows kcap).  Only the [C][U] hypothesis and cluster counts come back to the host."""
  x, offsets = _device_rows(tensors)
  device = x.device
  n, rows, configs = len(tensors), int(offsets[-1]), 1 if pairs is None else len(pairs)
  k = n_best or 1
  labels = torch.empty((configs, k, rows), dtype=torch.int32, device=device)
  scores = torch.empty((configs, max(n, 1), k), dtype=torch.float32, device=device)
  speakers = torch.empty((configs, max(n, 1), k), dtype=torch.int32, device=device)
  count = torch.empty((configs, max(n, 1)), dtype=torch.int32, device=device)
  stream = torch.cuda.current_stream(device).cuda_stream
  mx, mn = bounds

  def decode(kcap):
    model.predict_device_sweep(x.data_ptr(), offsets, labels.data_ptr(), scores.data_ptr(), pairs,
                               beam_size=args.beam_size, look_ahead=args.look_ahead,
                               test_iteration=args.test_iteration, kcap=kcap, stream=stream, max_speakers=mx,
                               min_speakers=mn, n_best=k, speakers_ptr=speakers.data_ptr(), count_ptr=count.data_ptr())
    model.stats()

  _grow_kcap(model, decode)
  labels = labels.to(torch.int64)
  counts = count[:, :n].cpu().numpy()
  spk0 = speakers[:, :n, 0].cpu().numpy()
  spans = [(int(offsets[u]), int(offsets[u + 1])) for u in range(n)]
  if n_best is None:
    hyps = [[labels[c, 0, a:b] for a, b in spans] for c in range(configs)]
  else:
    hyps = [[NBest(labels[c, :m, a:b], scores[c, u, :m], speakers[c, u, :m])
             for u, ((a, b), m) in enumerate(zip(spans, counts[c].tolist()))] for c in range(configs)]
  return hyps, spk0


def _decode_task(model, args, n_best, sequence, max_speakers, min_speakers):
  """One pool task of the CPU parallel_predict (module level: the pool pickles it): (hypotheses, speakers) of one
  sequence, as UISRNN._decode gives them."""
  bounds = tuple(None if b is None else np.array([b], np.int32) for b in (max_speakers, min_speakers))
  hyps, speakers = model._decode([sequence], args, bounds, n_best, None)  # pylint: disable=protected-access
  return hyps[0][0], speakers[0][0]


def _decode_shard(native_model, sequences, args, bounds, n_best, out, position):
  """One device's shard of the CUDA parallel_predict, run on its own host thread (the C ABI releases the GIL)."""
  out[position] = _native_decode(native_model(), sequences, args, bounds, n_best, None)


def _take(bound, indices):
  return bound[indices] if bound is not None else None


def parallel_predict(model, test_sequences, args, num_processes=4, *, max_speakers=None, min_speakers=None,
                     n_best=None):
  """Parallel prediction over a list of sequences (uisrnn.py:593-623).

  CPU model: a forkserver process pool, as the reference.  CUDA model: `num_processes` is the
  number of GPUs to use (capped by the visible devices); the list is split by total frame count
  and each shard is decoded by one native call on its own device, from its own host thread
  (the C ABI releases the GIL).  Utterances are independent, so there is no collective.
  Speaker bounds and n_best as in `UISRNN.predict`; per-utterance values travel with their shards.
  """
  if not isinstance(test_sequences, list):
    raise TypeError('test_sequences must be a list.')
  if n_best is not None:
    n_best = _check_n_best(n_best, args)
  bounds = _speaker_bounds(len(test_sequences), max_speakers, min_speakers)
  for sequence in test_sequences:
    _check_test_sequence(sequence, model.observation_dim)
  n = len(test_sequences)
  n_dev = max(1, min(int(num_processes), torch.cuda.device_count())) if model.device.type == 'cuda' else 0
  if n_dev == 1 or (n_dev and n < 2):
    hyps, speakers = model._decode(test_sequences, args, bounds, n_best, None)  # pylint: disable=protected-access
    hyps, speakers = hyps[0], speakers[0]
  elif n_dev:
    from . import native
    shards = shard_by_frames([len(s) for s in test_sequences], n_dev)
    weights = model.export_weights()
    makers = [functools.partial(model._native_model, 0)] + [  # pylint: disable=protected-access
        functools.partial(native.NativeModel, weights, device=d) for d in range(1, n_dev)]
    results, threads = [None] * n_dev, []
    for d, shard in enumerate(shards):
      thread = threading.Thread(target=_decode_shard, args=(
          makers[d], [test_sequences[i] for i in shard], args, (_take(bounds[0], shard), _take(bounds[1], shard)),
          n_best, results, d))
      thread.start()
      threads.append(thread)
    for thread in threads:
      thread.join()
    hyps, speakers = [None] * n, np.zeros(n, np.int32)
    for shard, result in zip(shards, results):
      if result is None:
        raise RuntimeError('parallel_predict: a device shard failed')
      for j, i in enumerate(shard):
        hyps[i], speakers[i] = result[0][0][j], result[1][0][j]
  else:
    ctx = multiprocessing.get_context('forkserver')
    model.rnn_model.share_memory()
    with ctx.Pool(num_processes) as pool:
      out = pool.starmap(functools.partial(_decode_task, model, args, n_best), zip(
          test_sequences, bounds[0] if bounds[0] is not None else [None] * n,
          bounds[1] if bounds[1] is not None else [None] * n))
    hyps, speakers = [o[0] for o in out], [o[1] for o in out]
  _warn_min_speakers([len(s) for s in test_sequences], [speakers], bounds[1], False, stacklevel=3)
  return hyps


def shard_columns(width, rank, world):
  """Columns of a (length-sorted) mini-batch owned by `rank` in data-parallel fit(): rank, rank + world,
  ... -- every shard stays sorted by decreasing length and the long sequences are spread evenly."""
  return np.arange(rank, width, world)


def shard_by_frames(lengths, n_shards):
  """Longest-processing-time-first partition of utterance indices into `n_shards` groups with
  near-equal total frame counts (cost of an utterance ~ its frame count).  Returns index lists."""
  order = sorted(range(len(lengths)), key=lambda i: -lengths[i])
  loads = [0] * n_shards
  shards = [[] for _ in range(n_shards)]
  for i in order:
    target = loads.index(min(loads))
    shards[target].append(i)
    loads[target] += lengths[i]
  for shard in shards:
    shard.sort()
  return shards
