"""Host-side data preparation for fit() and result reporting.

Behavioural mirror of `/root/reference/uisrnn/utils.py` (same function names, arguments, return
values, exceptions and -- where random numbers are drawn -- the same sequence of `random` /
`numpy.random` calls, so a seeded fit() sees the same batches as the reference).  The per-speaker
grouping is done with one factorisation + stable sort instead of one string comparison pass per
speaker (the reference's `np.where(cluster_id == i)` loop, utils.py:186-201, is O(#speakers x N)
on a string array and dominates short fits).
"""
import random
import string

import numpy as np
import torch

_ALPHABET = string.ascii_uppercase + string.digits


def generate_random_string(length=6):
  """Random upper-case/digit string; one `random.choice` per character (utils.py:24-35)."""
  return ''.join([random.choice(_ALPHABET) for _ in range(length)])


def enforce_cluster_id_uniqueness(cluster_ids):
  """Prefixes every label of sequence i with a fresh random id (utils.py:38-61)."""
  if not isinstance(cluster_ids, list):
    raise TypeError('cluster_ids must be a list')
  unique_ids = []
  for labels in cluster_ids:
    prefix = generate_random_string()
    if isinstance(labels, np.ndarray):
      labels = labels.tolist()
    if not isinstance(labels, list):
      raise TypeError('Elements of cluster_ids must be list or numpy.ndarray')
    unique_ids.append(['_'.join([prefix, label]) for label in labels])
  return unique_ids


def host_labels(cluster_ids):
  """`cluster_ids` with every integer torch tensor [N] replaced by the list of the strings str(v) of its values v: the
  label rule of a fit from tensors, under which such a tensor trains exactly as that list of strings does.  All the
  tensors are read back in one copy (8 bytes per label); other entries are returned as they are."""
  positions = [u for u, ids in enumerate(cluster_ids) if isinstance(ids, torch.Tensor)]
  if not positions:
    return cluster_ids
  for u in positions:
    ids = cluster_ids[u]
    if ids.dtype.is_floating_point or ids.dtype.is_complex or ids.dtype == torch.bool:
      raise TypeError('utterance {}: a label tensor must have an integer dtype, got {}'.format(u, ids.dtype))
    if ids.ndim != 1:
      raise ValueError('a label sequence must be a 1-D sequence of labels')
  # uint64 travels as its int64 bit pattern (a same-size view, any strides) and is unwrapped on the host
  values = torch.cat([cluster_ids[u].detach().view(torch.int64) if cluster_ids[u].dtype == torch.uint64 else
                      cluster_ids[u].detach().to(torch.int64) for u in positions]).cpu().tolist()
  out, start = list(cluster_ids), 0
  for u in positions:
    n = cluster_ids[u].shape[0]
    part = values[start:start + n]
    if cluster_ids[u].dtype == torch.uint64:
      part = [v + 2 ** 64 if v < 0 else v for v in part]
    out[u] = [str(v) for v in part]
    start += n
  return out


def concatenate_training_data(train_sequences, train_cluster_ids, enforce_uniqueness=True, shuffle=True):
  """Validates, optionally uniquifies + shuffles, then concatenates sequences (utils.py:64-123).

  Sequences that are torch tensors are not concatenated: the shuffled list of them is returned in place of the
  concatenated sequence (the device trainer reads their rows where they are), and their label sequences may be integer
  torch tensors, taken as host_labels defines them.  The `random` calls are the same either way.  With ndarray
  sequences the label sequences follow the reference's rules: a tensor among them is a TypeError."""
  if not isinstance(train_sequences, list) or not isinstance(train_cluster_ids, list):
    raise TypeError('train_sequences and train_cluster_ids must be lists')
  if len(train_sequences) != len(train_cluster_ids):
    raise ValueError('train_sequences and train_cluster_ids must have same size')
  tensors = any(isinstance(sequence, torch.Tensor) for sequence in train_sequences)
  if tensors:
    train_cluster_ids = host_labels(train_cluster_ids)
  train_cluster_ids = [ids.tolist() if isinstance(ids, np.ndarray) else ids for ids in train_cluster_ids]
  expected_dim = None
  for position, (sequence, ids) in enumerate(zip(train_sequences, train_cluster_ids)):
    length, dim = sequence.shape
    if position == 0:
      expected_dim = dim
    elif dim != expected_dim:
      raise ValueError('train_sequences must have consistent observation dimension')
    if not isinstance(ids, list):
      raise TypeError('Elements of train_cluster_ids must be list or numpy.ndarray')
    if len(ids) != length:
      raise ValueError('Each train_sequence and its train_cluster_id must have same length')
  if enforce_uniqueness:
    train_cluster_ids = enforce_cluster_id_uniqueness(train_cluster_ids)
  if shuffle:
    paired = list(zip(train_sequences, train_cluster_ids))
    random.shuffle(paired)
    train_sequences, train_cluster_ids = zip(*paired)
  if tensors:
    concatenated_sequence = list(train_sequences)
  else:
    concatenated_sequence = np.concatenate(train_sequences, axis=0)
  concatenated_ids = [label for ids in train_cluster_ids for label in ids]
  return concatenated_sequence, concatenated_ids


def _contiguous_runs(index_sequence):
  """Splits a sorted index array into maximal runs of consecutive integers."""
  index_sequence = np.asarray(index_sequence)
  if len(index_sequence) <= 1:
    return [index_sequence]
  breaks = np.flatnonzero(np.diff(index_sequence) != 1) + 1
  return np.split(index_sequence, breaks)


def sample_permuted_segments(index_sequence, number_samples):
  """`number_samples` copies of `index_sequence` with its contiguous runs randomly reordered;
  one `np.random.permutation(#runs)` per copy (utils.py:126-169)."""
  runs = _contiguous_runs(index_sequence)
  samples = []
  for _ in range(number_samples):
    order = np.random.permutation(len(runs))
    samples.append(np.concatenate([runs[i] for i in order]))
  return samples


def resize_sequence(sequence, cluster_id, num_permutations=None):
  """Regroups a concatenated sequence by speaker (utils.py:172-201).

  Returns `(sub_sequences, seq_lengths)`: one array per speaker (times `num_permutations` block
  permutations when > 1), speakers in `np.unique` order, and each length + 1.
  """
  index_lists, seq_lengths = resize_indices(cluster_id, num_permutations)
  return [sequence[indices, :] for indices in index_lists], seq_lengths


def resize_indices(cluster_id, num_permutations=None):
  """`resize_sequence` without the data: the ROW INDICES of every sub-sequence (same order, same
  `np.random.permutation` calls) and each length + 1.  The device-resident training path gathers rows
  by these indices instead of holding `num_permutations` float64 copies of the training set."""
  cluster_id = np.asarray(cluster_id)
  unique_ids, inverse = np.unique(cluster_id, return_inverse=True)
  order = np.argsort(inverse, kind='stable')          # indices grouped by speaker, ascending inside
  bounds = np.concatenate([[0], np.cumsum(np.bincount(inverse, minlength=len(unique_ids)))])
  sub_sequences, seq_lengths = [], []
  permute = bool(num_permutations) and num_permutations > 1
  for k in range(len(unique_ids)):
    indices = order[bounds[k]:bounds[k + 1]]
    if permute:
      for sampled in sample_permuted_segments(indices, num_permutations):
        sub_sequences.append(sampled)
        seq_lengths.append(len(indices) + 1)
    else:
      sub_sequences.append(indices)
      seq_lengths.append(len(indices) + 1)
  return sub_sequences, seq_lengths


class BatchSampler:
  """The draw of `pack_sequence` (utils.py:230-237) without building the batch: `draw()` makes the same
  `np.random.choice(num_clusters, batch_size)` call and returns the ids of the chosen sub-sequences in
  column order (lengths descending) with their lengths (+ 1 for the zero frame)."""

  def __init__(self, seq_lengths, batch_size):
    seq_lengths = np.asarray(seq_lengths)
    self.batch_size = batch_size
    self.sorted_lengths = np.sort(seq_lengths)[::-1]
    self.permute_index = np.argsort(seq_lengths)[::-1]

  def draw(self):
    count = len(self.sorted_lengths)
    chosen = np.arange(count) if self.batch_size is None else np.sort(np.random.choice(count, self.batch_size))
    return self.permute_index[chosen], self.sorted_lengths[chosen]


def pack_batch(sub_sequences, seq_lengths, batch_size, observation_dim):
  """The host half of `pack_sequence`: draws the batch (same `np.random.choice` call as
  utils.py:237) and returns `(rnn_input float64 [L, B, D] zero-padded time-major, lengths [B])`,
  lengths sorted descending and counting the leading zero frame."""
  seq_lengths = np.asarray(seq_lengths)
  num_clusters = len(seq_lengths)
  sorted_lengths = np.sort(seq_lengths)[::-1]
  permute_index = np.argsort(seq_lengths)[::-1]
  if batch_size is None:
    chosen = np.arange(num_clusters)
    width = num_clusters
  else:
    chosen = np.sort(np.random.choice(num_clusters, batch_size))
    width = batch_size
  lengths = sorted_lengths[chosen]
  rnn_input = np.zeros((lengths[0], width, observation_dim))
  for column, pick in enumerate(chosen):
    rnn_input[1:sorted_lengths[pick], column, :] = sub_sequences[permute_index[pick]]
  return rnn_input, np.ascontiguousarray(lengths)


def pack_sequence(sub_sequences, seq_lengths, batch_size, observation_dim, device):
  """Builds one training batch (utils.py:204-250): `np.random.choice(num_clusters, batch_size)`
  (with replacement) over the sub-sequences sorted by decreasing length, a zero frame prepended,
  zero padded to the longest, packed for the GRU.  Returns `(packed_rnn_input, rnn_truth)` with
  `rnn_truth = rnn_input[1:]`."""
  rnn_input, lengths = pack_batch(sub_sequences, seq_lengths, batch_size, observation_dim)
  rnn_input = torch.from_numpy(rnn_input).float().to(device)
  packed_rnn_input = torch.nn.utils.rnn.pack_padded_sequence(
      rnn_input, np.ascontiguousarray(lengths), batch_first=False)
  return packed_rnn_input, rnn_input[1:, :, :]


def output_result(model_args, training_args, test_record):
  """Formats and appends the experiment summary to `layer_<H>_<depth>_<dropout>_result.txt`
  (utils.py:253-285)."""
  accuracies = [accuracy for accuracy, _ in test_record]
  lines = [
      'Config:',
      '  sigma_alpha: {}'.format(training_args.sigma_alpha),
      '  sigma_beta: {}'.format(training_args.sigma_beta),
      '  crp_alpha: {}'.format(model_args.crp_alpha),
      '  learning rate: {}'.format(training_args.learning_rate),
      '  regularization: {}'.format(training_args.regularization_weight),
      '  batch size: {}'.format(training_args.batch_size),
      '',
      'Performance:',
      '  averaged accuracy: {:.6f}'.format(np.mean(accuracies)),
      '  accuracy numbers for all testing sequences:',
  ]
  output_string = '\n'.join(lines)
  for accuracy in accuracies:
    output_string += '\n    {:.6f}'.format(accuracy)
  output_string += '\n' + '=' * 80 + '\n'
  filename = 'layer_{}_{}_{:.1f}_result.txt'.format(
      model_args.rnn_hidden_size, model_args.rnn_depth, model_args.rnn_dropout)
  with open(filename, 'a') as handle:
    handle.write(output_string)
  return output_string


def estimate_transition_bias(cluster_ids, smooth=1):
  """Smoothed fraction of speaker changes (utils.py:288-313); returns `(bias, denominator)`."""
  transitions = smooth
  denominator = 2 * smooth
  for labels in cluster_ids:
    labels = np.asarray(list(labels) if isinstance(labels, str) else labels)
    if len(labels) > 1:
      transitions += int(np.count_nonzero(labels[:-1] != labels[1:]))
      denominator += len(labels) - 1
  return transitions / denominator, denominator
