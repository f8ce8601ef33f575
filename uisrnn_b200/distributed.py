"""Multi-process (one process per GPU) utterance sharding for predict().

The path shards naturally: every test utterance is an independent beam search (the reference
maps `predict_single` over the list, `/root/reference/uisrnn/uisrnn.py:587-589, 619-621`), so the
only cross-rank traffic is the gather of the label lists -- no data-path collective.  Works with
any `torch.distributed` backend (NCCL on the GPU box, gloo in the CPU tests).
"""
import numpy as np
import torch
import torch.distributed as dist

from . import native
from .uisrnn import _check_test_sequence, _warn_min_speakers, shard_by_frames


def predict_sharded(model, test_sequences, args, group=None, lengths=None, root=None, as_arrays=False, *,
                    max_speakers=None, min_speakers=None):
  """Every rank passes the same list; rank r decodes the r-th shard (longest-first partition by
  frame count) with `model.predict`, and every rank returns the complete, ordered result.

  `lengths` (optional): the frame counts of ALL utterances.  With it a rank only needs to hold the
  utterances of its own shard -- `test_sequences[i]` may be None (or a zero-argument callable that
  produces the array) for every other i -- so a large list is never materialised on every rank
  (`my_shard(lengths)` tells a rank which entries it owns).

  The labels travel as ONE int32 tensor per rank (all_gather / gather over NCCL when the model lives on a
  CUDA device, gloo otherwise), not as pickled Python lists.  `root=r`: only rank r receives the merged
  result (what the reference's `parallel_predict` caller gets, uisrnn.py:619-623); the other ranks return
  their own shard in place and None elsewhere.  `as_arrays=True`: entries are numpy int32 arrays instead of
  lists of Python ints (building Python ints costs ~10 ns per label in one thread, which at several million
  frames per second per GPU is the slowest stage of an 8-GPU job).

  `max_speakers` / `min_speakers`: speaker bounds as in `UISRNN.predict` (an int, or one value per utterance, which
  travels with its shard); each rank warns about the utterances of its own shard that fell short of min_speakers."""
  if not isinstance(test_sequences, list):
    raise TypeError('test_sequences must be a list.')
  if lengths is not None and len(lengths) != len(test_sequences):
    raise ValueError('lengths must have one entry per test sequence.')
  bounds = native.speaker_bounds(len(test_sequences), max_speakers, min_speakers)
  if not (dist.is_available() and dist.is_initialized()):
    return _decode_labels(model, [_materialise(s) for s in test_sequences], args, range(len(test_sequences)), bounds,
                          as_arrays)
  world = dist.get_world_size(group)
  rank = dist.get_rank(group)
  lengths = [len(s) for s in test_sequences] if lengths is None else [int(n) for n in lengths]
  shards = shard_by_frames(lengths, world)
  mine = _decode_labels(model, [_materialise(test_sequences[i]) for i in shards[rank]], args, shards[rank], bounds,
                        True) if shards[rank] else []
  counts = [sum(lengths[i] for i in shard) for shard in shards]
  use_cuda = getattr(model, 'device', None) is not None and model.device.type == 'cuda' and \
      dist.get_backend(group) == 'nccl'
  device = model.device if use_cuda else torch.device('cpu')
  flat = np.concatenate(mine).astype(np.int32, copy=False) if mine else np.zeros(0, np.int32)
  assert flat.size == counts[rank]
  width = max(max(counts), 1)
  send = torch.zeros(width, dtype=torch.int32, device=device)   # equal-sized pieces: pad to the largest shard
  send[:flat.size] = torch.from_numpy(flat).to(device)
  receives = rank == root or root is None
  if root is None:
    recv = [torch.empty(width, dtype=torch.int32, device=device) for _ in range(world)]
    dist.all_gather(recv, send, group=group)
  else:
    recv = [torch.empty(width, dtype=torch.int32, device=device) for _ in range(world)] if rank == root else None
    dist.gather(send, recv, dst=root, group=group)
  merged = [None] * len(test_sequences)
  if receives:
    for shard, piece, count in zip(shards, recv, counts):
      flat_r = piece[:count].cpu().numpy()
      pos = 0
      for i in shard:
        merged[i] = flat_r[pos:pos + lengths[i]]
        pos += lengths[i]
  else:
    for i, lab in zip(shards[rank], mine):
      merged[i] = lab
  if not as_arrays:
    merged = [m.tolist() if m is not None else None for m in merged]
  return merged


def _decode_labels(model, sequences, args, indices, bounds, as_arrays):
  """Hypothesis 0's labels of `sequences` (int32 arrays with as_arrays), one warning for those that fell short of
  min_speakers.  `indices`: the positions of `sequences` in the caller's list; `bounds`: speaker bounds over that whole
  list (None = absent)."""
  for sequence in sequences:
    _check_test_sequence(sequence, model.observation_dim)  # the reference's TypeError / ValueError sites
  indices = list(indices)
  mine = tuple(b[indices] if b is not None else None for b in bounds)
  hyps, speakers = model._decode(sequences, args, mine, None, None, as_arrays)  # pylint: disable=protected-access
  _warn_min_speakers([len(s) for s in sequences], speakers, mine[1], False, stacklevel=4, indices=indices)
  return [np.asarray(lab, np.int32) for lab in hyps[0]] if as_arrays else hyps[0]


def my_shard(lengths, group=None):
  """Indices of the utterances this rank decodes in `predict_sharded(..., lengths=lengths)`."""
  if not (dist.is_available() and dist.is_initialized()):
    return list(range(len(lengths)))
  return shard_by_frames(list(lengths), dist.get_world_size(group))[dist.get_rank(group)]


def _materialise(entry):
  if callable(entry):
    entry = entry()
  if entry is None:
    raise ValueError('predict_sharded: an utterance of this rank\'s shard is missing (None).')
  return entry
