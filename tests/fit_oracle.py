"""Float64 oracle of one fit() iteration -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The reference's formulation of a training iteration (uisrnn.py:252-295 of the reference; uisrnn_b200/uisrnn.py
fit_concatenated) evaluated with autograd in a chosen dtype, from the same inputs the device trainer takes
(uis_trainer_step): parameters in native.param_order(depth), a time-major zero-padded batch x [L, B, D] whose row 0
is the zero frame, and lengths sorted descending with lengths[0] == L.  The packed GRU, the MLP, the running mean over
time, the masked weighted MSE, the sigma^2 prior and the per-tensor norm regulariser; with dropout scales given, the
stacked GRU runs layer by layer and the output of layer l is multiplied by scales[l] before layer l + 1 sees it
(what nn.GRU(dropout=p) does in train mode, with the trainer's masks instead of PyTorch's).

In float64 on the CPU (or on a GPU with cuDNN off) neither TF32 nor cuDNN is involved, so the result is the exact
value of the operation up to float64 rounding: the yardstick the fp32 kernels of csrc/uis_train.cu are pinned to by
tests/test_gpu_fit_fp64.py, and in data-parallel mode (shard_dropout_scales) by tests/test_gpu_fit_dp_fp64.py.
tests/test_fit_oracle_cpu.py pins this module to the repository's own torch fit() path.

FitAdam is the tail of the iteration: clip_grad_norm_ over rnn_model.parameters(), torch.optim.Adam with its defaults
(the param groups of UISRNN._get_optimizer) and the sigma^2 clamp, with its own float64 state, driven by gradients the
caller supplies.
"""
import contextlib

import numpy as np
import torch
from torch import nn

from uisrnn_b200 import native

_KINDS = ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh')


def depth_of(params):
  return sum(1 for k in params if k.startswith('gru.weight_ih_l'))


def rnn_names(depth):
  """The tensors of rnn_model.parameters(), in its order: regularised one by one and clipped as a group."""
  return native.param_order(depth)[:-2]


def dropout_scales(seed, iteration, depth, L, B, H, p):
  """Multipliers of the outputs of layers 0..depth-2 in training iteration `iteration` of a trainer created with
  dropout_seed=seed, rnn_dropout=p: keep / (1 - p) with the trainer's keep masks (native.dropout_keep_mask) and its
  fp32 scale 1 / (1 - p).  Float64 arrays [L, B, H]."""
  inv_keep = float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))
  return [native.dropout_keep_mask(seed, iteration, l, L * B * H, p).reshape(L, B, H) * inv_keep
          for l in range(depth - 1)]


def shard_dropout_scales(seeds, iteration, depth, lengths, H, p, world):
  """dropout_scales of a data-parallel iteration, laid out on the full batch: rank r (trainer seed seeds[r]) holds
  columns shard_columns(B, r, world) and masks them as its own zero-padded shard [L_r, B_r, H], L_r the length of
  its first column.  Column b, the j-th of rank r, carries dropout_scales(seeds[r], iteration, depth, L_r, B_r, H,
  p)[:, j] at rows < L_r and zeros below (padding of every rank's layout).  Without dropout, the all-reduced
  iteration is the full-batch one, so these scales make losses_and_grads on the full batch the oracle of every
  rank's step.  Float64 arrays [L, B, H]."""
  from uisrnn_b200.uisrnn import shard_columns
  lengths = np.asarray(lengths)
  L, B = int(lengths[0]), len(lengths)
  out = [np.zeros((L, B, H)) for _ in range(depth - 1)]
  for r in range(world):
    mine = shard_columns(B, r, world)
    if not len(mine):
      continue
    Lr = int(lengths[mine[0]])
    for full, shard in zip(out, dropout_scales(seeds[r], iteration, depth, Lr, len(mine), H, p)):
      full[:Lr, mine] = shard
  return out


def random_params(D, H, depth, seed):
  """Parameters as a fresh model draws them (nn.GRU / nn.Linear: U(-1/sqrt(fan), 1/sqrt(fan))), with
  rnn_init_hidden ~ N(0, 0.1) and sigma2 ~ U(0.05, 0.2) so that neither is a constant; float32 values."""
  rng = np.random.default_rng(seed)
  u = lambda shape, fan: rng.uniform(-1, 1, shape) / np.sqrt(fan)
  p = {}
  for l in range(depth):
    p['gru.weight_ih_l%d' % l] = u((3 * H, D if l == 0 else H), H)
    p['gru.weight_hh_l%d' % l] = u((3 * H, H), H)
    p['gru.bias_ih_l%d' % l] = u(3 * H, H)
    p['gru.bias_hh_l%d' % l] = u(3 * H, H)
  p['linear_mean1.weight'] = u((H, H), H)
  p['linear_mean1.bias'] = u(H, H)
  p['linear_mean2.weight'] = u((D, H), H)
  p['linear_mean2.bias'] = u(D, H)
  p['rnn_init_hidden'] = rng.normal(0, 0.1, depth * H)
  p['sigma2'] = rng.uniform(0.05, 0.2, D)
  return {k: np.asarray(p[k], np.float32) for k in native.param_order(depth)}


def make_batch(lengths, D, seed, zeros=False):
  """A batch as utils.pack_batch lays it out: x [L, B, D] float32, x[0] the zero frame, zero padding; column b
  holds lengths[b] - 1 frames around a per-column mean (sub-sequences of one speaker), none of them zero.
  zeros=True also plants exact zeros in real frames -- single features, dimension 0 included, and one whole frame."""
  lengths = np.asarray(lengths, np.int32)
  L, B = int(lengths[0]), len(lengths)
  assert np.all(np.diff(lengths) <= 0) and lengths[-1] >= 1
  rng = np.random.default_rng(seed)
  x = rng.normal(0, 0.3, (L, B, D)) + rng.normal(0, 1, (1, B, D))
  x[np.abs(x) < 1e-3] = 1e-3
  x[0] = 0
  for b, n in enumerate(lengths):
    x[n:, b] = 0
  if zeros:
    real = [(t, b) for b in range(B) for t in range(1, int(lengths[b]))]
    for i in rng.choice(len(real), max(1, len(real) // 4), replace=False):
      t, b = real[i]
      x[t, b, rng.integers(0, D)] = 0
    for i in rng.choice(len(real), max(1, len(real) // 8), replace=False):
      t, b = real[i]
      x[t, b, 0] = 0
    t, b = real[len(real) // 2]
    x[t, b] = 0
  return x.astype(np.float32), lengths


def _no_cudnn(device):
  return torch.backends.cudnn.flags(enabled=False) if torch.device(device).type == 'cuda' else contextlib.nullcontext()


def weighted_mse_loss(input_tensor, target_tensor, weight):
  """loss_func.weighted_mse_loss without its cast of the weight to float32: the same formula in the dtype of the
  operands."""
  dim = input_tensor.size()[-1]
  squared = ((input_tensor - target_tensor) ** 2).view(-1, dim)
  rows = float(squared.size()[0])
  non_zero_rows = torch.sum(squared[:, 0] != 0).to(squared.dtype)
  return torch.mean(squared * weight.view(-1)) * weight.nelement() * rows / non_zero_rows


def losses_and_grads(params, x, lengths, hp, scales=None, dtype=torch.float64, device='cpu'):
  """One iteration's losses and gradients.

  params: dict name -> array in native.param_order(depth) (rnn_init_hidden flattened to [depth * H]);
  x: [L, B, D] batch as uis_trainer_step takes it; lengths: [B]; hp: dict with sigma_alpha, sigma_beta and
  regularization_weight; scales: None, or the depth - 1 dropout multipliers of dropout_scales().
  Returns ((loss1, loss2, loss3), grads): python floats and a dict name -> float64 array shaped as params[name].
  The gradients are those of loss1 + loss2 + loss3 (the regulariser included), before clipping."""
  depth = depth_of(params)
  H = np.asarray(params['linear_mean1.weight']).shape[0]
  t = {k: nn.Parameter(torch.tensor(np.asarray(v, np.float64), dtype=dtype, device=device)) for k, v in params.items()}
  xt = torch.tensor(np.asarray(x, np.float64), dtype=dtype, device=device)
  L, B, D = xt.shape
  lengths = [int(v) for v in lengths]
  h0 = t['rnn_init_hidden'].view(depth, 1, H)
  with _no_cudnn(device):
    if scales is None:
      gru = nn.GRU(D, H, depth).to(device=device, dtype=dtype)
      for l in range(depth):
        for kind in _KINDS:
          setattr(gru, '{}_l{}'.format(kind, l), t['gru.{}_l{}'.format(kind, l)])
      packed = nn.utils.rnn.pack_padded_sequence(xt, lengths)
      out, _ = gru(packed, h0.repeat(1, B, 1))
      out, _ = nn.utils.rnn.pad_packed_sequence(out, total_length=L)
    else:
      assert len(scales) == depth - 1
      out = xt
      for l in range(depth):
        gru = nn.GRU(D if l == 0 else H, H, 1).to(device=device, dtype=dtype)
        for kind in _KINDS:
          setattr(gru, kind + '_l0', t['gru.{}_l{}'.format(kind, l)])
        if l > 0:
          out = out * torch.tensor(scales[l - 1], dtype=dtype, device=device)
        out, _ = gru(nn.utils.rnn.pack_padded_sequence(out, lengths), h0[l:l + 1].repeat(1, B, 1))
        out, _ = nn.utils.rnn.pad_packed_sequence(out, total_length=L)
  a1 = torch.relu(out @ t['linear_mean1.weight'].T + t['linear_mean1.bias'])
  mean = a1 @ t['linear_mean2.weight'].T + t['linear_mean2.bias']
  steps = torch.arange(1, L + 1, device=device, dtype=dtype)
  mean = torch.cumsum(mean, dim=0) * (1.0 / steps).view(-1, 1, 1)
  truth = xt[1:]
  mask = (truth != 0).to(dtype)
  sigma2 = t['sigma2']
  loss1 = weighted_mse_loss(mask * mean[:-1], truth, 1 / (2 * sigma2))
  res = ((mask * mean[:-1] - truth) ** 2).view(-1, D)
  nnz = torch.sum((res != 0).to(dtype), dim=0)
  loss2 = ((2 * hp['sigma_alpha'] + nnz + 2) / (2 * nnz) * torch.log(sigma2)).sum() + \
      (hp['sigma_beta'] / (sigma2 * nnz)).sum()
  loss3 = hp['regularization_weight'] * sum(torch.norm(t[k]) for k in rnn_names(depth))
  (loss1 + loss2 + loss3).backward()
  grads = {k: v.grad.detach().cpu().numpy().astype(np.float64).reshape(np.shape(params[k])) for k, v in t.items()}
  return (float(loss1.detach()), float(loss2.detach()), float(loss3.detach())), grads


class FitAdam:
  """clip_grad_norm_(rnn_model.parameters(), grad_max_norm) + torch.optim.Adam (defaults, lr = learning_rate) over
  the param groups of UISRNN._get_optimizer (sigma2 only when train_sigma2) + sigma2.clamp_(min=1e-6), in float64.

  step(grads, params=None): applies one step to the oracle's own parameters, or first loads `params` into them
  (so that a test can drive the optimiser from the device trainer's parameters and gradients of every step while
  the Adam moments stay the oracle's).  Returns the new parameters (float64, shaped as given); the clip coefficient
  of the step is in .clip_coef."""

  def __init__(self, params, hp):
    self.depth = depth_of(params)
    self.hp = hp
    self.shapes = {k: np.shape(v) for k, v in params.items()}
    self.t = {k: nn.Parameter(torch.tensor(np.asarray(v, np.float64), dtype=torch.float64)) for k, v in params.items()}
    groups = [{'params': [self.t[k] for k in rnn_names(self.depth)]}, {'params': [self.t['rnn_init_hidden']]}]
    if hp['train_sigma2']:
      groups.append({'params': [self.t['sigma2']]})
    self.opt = torch.optim.Adam(groups, lr=hp['learning_rate'])
    self.clip_coef = None

  def step(self, grads, params=None):
    with torch.no_grad():
      if params is not None:
        for k, v in params.items():
          self.t[k].copy_(torch.tensor(np.asarray(v, np.float64).reshape(self.shapes[k])))
      for k, v in grads.items():
        self.t[k].grad = torch.tensor(np.asarray(v, np.float64).reshape(self.shapes[k]))
    norm = float(nn.utils.clip_grad_norm_([self.t[k] for k in rnn_names(self.depth)], self.hp['grad_max_norm']))
    self.clip_coef = min(self.hp['grad_max_norm'] / (norm + 1e-6), 1.0)
    self.opt.step()
    with torch.no_grad():
      self.t['sigma2'].clamp_(min=1e-6)
    return self.parameters()

  def parameters(self):
    return {k: v.detach().numpy().copy() for k, v in self.t.items()}
