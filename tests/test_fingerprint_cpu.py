"""UISRNN._fingerprint, the key that decides when the device twin of a model (its weights, tensor-core planes and
scales on the GPU) is rebuilt: exact on every parameter, including edits through `.data` that keep `_version` and
every |value|.  CPU only."""
import numpy as np
import pytest
import torch

from helpers import load_weights, uisrnn_from_weights


@pytest.fixture
def model():
  return uisrnn_from_weights(load_weights('model_small.npz'))


def params(m):
  return dict(m.rnn_model.named_parameters(), rnn_init_hidden=m.rnn_init_hidden, sigma2=m.sigma2)


def test_unchanged_parameters_keep_the_key(model):
  before = model._fingerprint()  # pylint: disable=protected-access
  assert model._fingerprint() == before  # pylint: disable=protected-access
  assert model._fingerprint(copy=False) == before  # pylint: disable=protected-access
  model.predict(np.zeros((3, 64)) + 0.1, __import__('helpers').inference_args(test_iteration=1))
  assert model._fingerprint(copy=False) == before  # pylint: disable=protected-access


@pytest.mark.parametrize('name', ['linear_mean2.weight', 'linear_mean1.weight', 'gru.weight_hh_l0', 'linear_mean1.bias',
                                  'rnn_init_hidden', 'sigma2'])
@pytest.mark.parametrize('edit', ['neg_row', 'swap_rows'])
def test_edits_through_data_change_the_key(model, name, edit):
  """A sign flip or a swap of two rows keeps `_version`, the L1 and L2 norms, and (before) the key."""
  p = params(model)[name]
  # rows of a matrix; the two halves of a vector (or of rnn_init_hidden [1, 1, H])
  d = p.data.view(-1, p.shape[-1]) if p.numel() > p.shape[-1] else p.data.view(2, -1)
  assert not torch.equal(d[0], d[1]) and bool((d[1] != 0).any())
  version = p._version  # pylint: disable=protected-access
  before = model._fingerprint()  # pylint: disable=protected-access
  norms = torch.stack([p.detach().double().norm(1), p.detach().double().norm(2)])
  if edit == 'neg_row':
    d[1].neg_()
  else:
    d[[0, 1]] = d[[1, 0]].clone()
  assert p._version == version  # pylint: disable=protected-access
  if edit == 'swap_rows':  # the same multiset of values
    assert torch.equal(torch.stack([p.detach().double().norm(1), p.detach().double().norm(2)]), norms)
  assert model._fingerprint() != before  # pylint: disable=protected-access
  assert model._fingerprint(copy=False) != before  # pylint: disable=protected-access


def test_nan_parameter_never_matches(model):
  model.sigma2.data[0] = float('nan')
  key = model._fingerprint()  # pylint: disable=protected-access
  assert key != key and model._fingerprint(copy=False) != key  # pylint: disable=protected-access


def test_scalars_and_shapes_are_part_of_the_key(model):
  before = model._fingerprint()  # pylint: disable=protected-access
  model.crp_alpha = model.crp_alpha * 2
  assert model._fingerprint(copy=False) != before  # pylint: disable=protected-access
  model.crp_alpha = model.crp_alpha / 2
  assert model._fingerprint(copy=False) == before  # pylint: disable=protected-access
  model.rnn_init_hidden = torch.nn.Parameter(model.rnn_init_hidden.detach().reshape(1, -1))
  assert model._fingerprint(copy=False) != before  # pylint: disable=protected-access
