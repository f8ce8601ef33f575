"""tests/fit_oracle.py (the float64 oracle of a fit() iteration that the device trainer is pinned to) against the
repository's own torch fit() arithmetic on the CPU: in float32 it computes what that path computes, in float64 it
differs from it by float32 rounding only, and its layer-by-layer dropout path with all-ones scales is the plain
stacked GRU."""
import numpy as np
import pytest

import fit_oracle

HP = {'sigma_alpha': 1.0, 'sigma_beta': 1.0, 'regularization_weight': 1e-5}


def _cpu_model(params, D, H, depth):
  import torch
  import uisrnn
  m, _, _ = uisrnn.parse_arguments([])
  m.observation_dim, m.rnn_hidden_size, m.rnn_depth, m.rnn_dropout, m.verbosity = D, H, depth, 0.0, 0
  m.enable_cuda = False
  model = uisrnn.UISRNN(m)
  assert model.device.type == 'cpu'
  model.rnn_model.load_state_dict({k: torch.from_numpy(params[k]) for k in fit_oracle.rnn_names(depth)})
  model.rnn_model.train()
  with torch.no_grad():
    model.rnn_init_hidden.copy_(torch.from_numpy(params['rnn_init_hidden']).view(depth, 1, H))
    model.sigma2.copy_(torch.from_numpy(params['sigma2']))
  return model


def _row_err(got, want):
  """Worst |got - want| over rows of 2-D tensors (whole tensor for 1-D), relative to the row's largest |want|."""
  got, want = np.atleast_2d(got), np.atleast_2d(want)
  scale = np.max(np.abs(want), axis=1, keepdims=True) + 1e-30
  return float(np.max(np.abs(got - want) / scale))


@pytest.mark.parametrize('D,H,depth', [(6, 8, 1), (5, 12, 2)])
def test_float32_oracle_equals_the_torch_fit_path(D, H, depth):
  import torch
  import uisrnn
  from test_gpu_fit import _torch_losses_and_grads
  params = fit_oracle.random_params(D, H, depth, seed=3 + depth)
  x, lengths = fit_oracle.make_batch([9, 9, 7, 4, 2], D, seed=5, zeros=True)
  model = _cpu_model(params, D, H, depth)
  _, targs, _ = uisrnn.parse_arguments([])
  want_losses, want = _torch_losses_and_grads(model, targs, x, lengths)
  got_losses, got = fit_oracle.losses_and_grads(params, x, lengths, HP, dtype=torch.float32)
  np.testing.assert_allclose(got_losses, want_losses, rtol=1e-6)
  assert set(got) == set(want)
  for k in want:
    assert _row_err(got[k], want[k].reshape(got[k].shape)) < 1e-6, k


@pytest.mark.parametrize('D,H,depth', [(6, 8, 1), (5, 12, 3)])
def test_float64_differs_from_float32_by_rounding_only(D, H, depth):
  import torch
  params = fit_oracle.random_params(D, H, depth, seed=7)
  x, lengths = fit_oracle.make_batch([12, 10, 10, 6, 3, 2], D, seed=8, zeros=True)
  l64, g64 = fit_oracle.losses_and_grads(params, x, lengths, HP)
  l32, g32 = fit_oracle.losses_and_grads(params, x, lengths, HP, dtype=torch.float32)
  np.testing.assert_allclose(l32, l64, rtol=1e-5)
  assert l32 != l64   # the float64 path does not round to float32 on the way
  for k in g64:
    assert g64[k].dtype == np.float64
    assert _row_err(g32[k], g64[k]) < 1e-4, k


@pytest.mark.parametrize('depth', [2, 3, 4])
def test_dropout_path_with_unit_scales_is_the_stacked_gru(depth):
  D, H = 4, 6
  params = fit_oracle.random_params(D, H, depth, seed=9)
  x, lengths = fit_oracle.make_batch([7, 6, 6, 2], D, seed=10)
  want_losses, want = fit_oracle.losses_and_grads(params, x, lengths, HP)
  ones = [np.ones((7, 4, H))] * (depth - 1)
  got_losses, got = fit_oracle.losses_and_grads(params, x, lengths, HP, scales=ones)
  assert got_losses == want_losses
  for k in want:
    assert np.array_equal(got[k], want[k]), k
  # and the scales do reach the upper layers
  drop = fit_oracle.dropout_scales(0x1234, 0, depth, 7, 4, H, 0.3)
  assert all(0.5 < (s > 0).mean() < 0.9 for s in drop)
  _, dropped = fit_oracle.losses_and_grads(params, x, lengths, HP, scales=drop)
  assert not np.array_equal(dropped['gru.weight_ih_l%d' % (depth - 1)], want['gru.weight_ih_l%d' % (depth - 1)])


def test_shard_dropout_scales_at_world_1_are_the_full_batch_scales():
  lengths, H, depth, p = [9, 7, 7, 4, 2], 5, 3, 0.3
  got = fit_oracle.shard_dropout_scales([0xABC], 2, depth, lengths, H, p, 1)
  want = fit_oracle.dropout_scales(0xABC, 2, depth, 9, 5, H, p)
  assert len(got) == depth - 1
  for g, w in zip(got, want):
    assert np.array_equal(g, w)


@pytest.mark.parametrize('world', [2, 3])
def test_shard_dropout_scales_follow_each_ranks_own_layout(world):
  """Column b of rank r = b % world carries the keep mask of element (t, j, h) of r's shard [L_r, B_r, H] (j = b //
  world, the column's place in that shard) under r's seed, for t < L_r; zeros below.  Seeds differ per rank, the
  first column of rank 1 is shorter than the batch, and rank 2 of world 3 has one column fewer than rank 0."""
  from uisrnn_b200 import native
  lengths, H, depth, p, it = [11, 8, 8, 6, 5, 3, 2, 2], 4, 3, 0.4, 5
  seeds = [0x1234 + 97 * r for r in range(world)]
  got = fit_oracle.shard_dropout_scales(seeds, it, depth, lengths, H, p, world)
  inv_keep = 1.0 / (1.0 - p)
  B = len(lengths)
  for l in range(depth - 1):
    assert got[l].shape == (11, B, H)
    for b in range(B):
      r, j = b % world, b // world
      Br = len(range(r, B, world))
      Lr = lengths[r]
      keep = native.dropout_keep_mask(seeds[r], it, l, Lr * Br * H, p).reshape(Lr, Br, H)[:, j]
      np.testing.assert_allclose(got[l][:Lr, b], keep * inv_keep, rtol=1e-6)
      assert np.array_equal(got[l][:Lr, b] > 0, keep)
      assert not got[l][Lr:, b].any()
  # the shards' masks are not one mask: rank 1's columns differ from what rank 0's seed would give them
  keep0 = native.dropout_keep_mask(seeds[0], it, 0, 11 * B * H, p).reshape(11, B, H)
  assert not np.array_equal(got[0][:lengths[1], 1] > 0, keep0[:lengths[1], 1])


def test_adam_matches_torch_optimizer_on_the_model():
  """FitAdam = clip_grad_norm_ + UISRNN._get_optimizer('adam') + clamp, applied to the same gradients."""
  import torch
  D, H, depth = 5, 8, 2
  params = fit_oracle.random_params(D, H, depth, seed=11)
  hp = dict(HP, learning_rate=1e-2, grad_max_norm=0.05, train_sigma2=True)
  model = _cpu_model({k: v.astype(np.float32) for k, v in params.items()}, D, H, depth)
  model.rnn_model.double()
  model.rnn_init_hidden.data = model.rnn_init_hidden.data.double()
  model.sigma2.data = model.sigma2.data.double()
  opt = model._get_optimizer('adam', hp['learning_rate'])  # pylint: disable=protected-access
  oracle = fit_oracle.FitAdam(params, hp)
  rng = np.random.default_rng(12)
  named = dict(model.rnn_model.named_parameters(), rnn_init_hidden=model.rnn_init_hidden, sigma2=model.sigma2)
  for _ in range(4):
    grads = {k: rng.normal(0, 1, np.shape(v)) for k, v in params.items()}
    for k, p in named.items():
      p.grad = torch.tensor(grads[k]).view(p.shape)   # a copy: clip_grad_norm_ scales it in place
    torch.nn.utils.clip_grad_norm_(model.rnn_model.parameters(), hp['grad_max_norm'])
    opt.step()
    model.sigma2.data.clamp_(min=1e-6)
    got = oracle.step(grads)
    assert oracle.clip_coef < 1
    for k, p in named.items():
      assert np.array_equal(got[k], p.detach().numpy().reshape(got[k].shape)), k
