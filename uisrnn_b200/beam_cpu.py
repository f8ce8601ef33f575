"""CPU beam search used when the caller explicitly selects the CPU device
(`--enable_cuda=False`, or no CUDA device present -- the reference's own device rule,
`/root/reference/uisrnn/uisrnn.py:90-91`).  It is NOT a fallback for the CUDA path: when the model
lives on a CUDA device, `UISRNN.predict` goes through libuisrnn_b200.so or raises.

Semantics follow `/root/reference/uisrnn/uisrnn.py:388-477, 523-561` (any depth, any look_ahead)
with the redundant network evaluations removed: the last look-ahead sub-step of a candidate is
scored without running the GRU (its result never enters the score), and
`CoreRNN(zeros, rnn_init_hidden)` is evaluated once per call instead of once per candidate.
"""
import numpy as np
import torch

from . import loss_func


def nbest_ranks(clusters, min_speakers, n_best):
  """Final ranks an N-best decode returns, given the cluster count of every final rank: the first `n_best` ranks
  with at least `min_speakers` clusters, or rank 0 alone when there is none."""
  return [r for r, k in enumerate(clusters) if k >= min_speakers][:n_best] or [0]


class _Hypothesis:
  """One beam entry: per-cluster running means / hidden states / visit and block counts."""
  __slots__ = ('means', 'hiddens', 'visits', 'blocks', 'trace', 'score', 'loss')  # loss: the last step's increment

  def __init__(self, parent=None):
    if parent is None:
      self.means, self.hiddens, self.visits, self.blocks, self.trace = [], [], [], [], []
      self.score = 0
    else:
      self.means = list(parent.means)
      self.hiddens = list(parent.hiddens)
      self.visits = list(parent.visits)
      self.blocks = list(parent.blocks)
      self.trace = list(parent.trace)
      self.score = parent.score


class CpuBeamSearch:
  """Decoder bound to one UISRNN model (weights are read at construction).  crp_alpha / transition_bias, when given,
  replace the model's values (a decoding-parameter sweep); the model is not changed."""

  def __init__(self, model, crp_alpha=None, transition_bias=None):
    self.rnn = model.rnn_model
    self.device = model.device
    p0 = model.transition_bias if transition_bias is None else transition_bias
    self.alpha = model.crp_alpha if crp_alpha is None else crp_alpha
    self.log_p0 = np.log(p0)
    self.log_1mp0 = np.log(1 - p0)
    self.log_alpha = np.log(self.alpha)
    self.rnn.eval()  # (mean0 / hidden0 below: no dropout between stacked layers, as in decode)
    with torch.no_grad():
      self.weight = (1 / (2 * model.sigma2)).detach()
      zeros = torch.zeros(1, 1, model.observation_dim, device=self.device)
      mean0, self.hidden0 = self.rnn(zeros, model.rnn_init_hidden.detach())
      self.mean0 = mean0.reshape(-1)

  def _mse(self, mean, frame):
    return loss_func.weighted_mse_loss(mean, frame, self.weight).cpu().numpy()

  def _advance(self, hyp, frame, cluster, update_state):
    """Applies one (frame, cluster) decision to `hyp` in place; False if the index is invalid."""
    count = len(hyp.means)
    if cluster > count:
      hyp.score = float('inf')
      return False
    total_blocks = sum(hyp.blocks)
    if cluster < count:
      previous = hyp.trace[-1]
      loss = self._mse(hyp.means[cluster], frame)
      if cluster == previous:
        loss -= self.log_1mp0
      else:
        loss -= self.log_p0 + np.log(hyp.blocks[cluster]) - np.log(total_blocks + self.alpha)
      if update_state:
        mean, hidden = self.rnn(frame.view(1, 1, -1), hyp.hiddens[cluster])
        seen = float(hyp.visits[cluster])
        hyp.means[cluster] = (hyp.means[cluster] * (seen - 1.0) + mean.reshape(-1)) / seen
        hyp.hiddens[cluster] = hidden
        hyp.visits[cluster] += 1
        if cluster != previous:
          hyp.blocks[cluster] += 1
        hyp.trace.append(cluster)
    else:
      loss = self._mse(self.mean0, frame)
      loss -= self.log_p0 + self.log_alpha - np.log(total_blocks + self.alpha)
      if update_state:
        mean, hidden = self.rnn(frame.view(1, 1, -1), self.hidden0)
        hyp.means.append(mean.reshape(-1))
        hyp.hiddens.append(hidden)
        hyp.visits.append(1)
        hyp.blocks.append(1)
        hyp.trace.append(cluster)
    hyp.loss = loss
    hyp.score = hyp.score + loss  # int 0 at first, float32 afterwards, as in the reference
    return True

  def _expand(self, hyp, frames, clusters):
    child = _Hypothesis(hyp)
    for frame, cluster in zip(frames, clusters):
      if not self._advance(child, frame, int(cluster), True):
        break
    return child

  def _score_table(self, hyp, frames, max_speakers=0):
    depth = frames.shape[0]
    count = len(hyp.means)
    table = np.full([count + 1 + i for i in range(depth)], np.inf)

    def walk(state, level, prefix):
      last = level == depth - 1
      for cluster in range(table.shape[level]):
        if max_speakers and cluster >= len(state.means) >= max_speakers:
          continue  # would open a cluster past max_speakers: the whole sub-tree stays +inf
        child = _Hypothesis(state)
        if not self._advance(child, frames[level], cluster, not last):
          continue
        if last:
          table[prefix + (cluster,)] = child.score
        else:
          walk(child, level + 1, prefix + (cluster,))

    walk(hyp, 0, ())
    return table

  @torch.no_grad()
  def score(self, sequence, labels):
    """(neg_likelihood, float32 [N] per-frame increments) of the trace that assigns frame t of `sequence` (float64
    [N, D]) to cluster labels[t] (canonical ids: 0, 1, 2, ... in order of first appearance): `_advance` with the state
    update, frame by frame from an empty hypothesis.  No test_iteration tiling."""
    self.rnn.eval()
    frames = torch.from_numpy(np.asarray(sequence)).float().to(self.device)
    hyp = _Hypothesis()
    increments = np.zeros(len(frames), np.float32)
    for t, (frame, cluster) in enumerate(zip(frames, labels)):
      if not self._advance(hyp, frame, int(cluster), True):
        raise ValueError('frame %d: label %d is not canonical' % (t, int(cluster)))
      increments[t] = hyp.loss
    return np.float32(hyp.score), increments

  @torch.no_grad()
  def decode(self, sequence, beam_size, look_ahead, test_iteration, max_speakers=0, min_speakers=0,
             return_speakers=False, n_best=None):
    """`sequence`: float64 [N, D] ndarray.  Returns the N labels of the last tiled copy (and, with
    return_speakers, the cluster count of the returned hypothesis).

    n_best=k: returns (labels, scores, clusters) of up to k final hypotheses instead (`nbest_ranks`): their
    labels of the last tiled copy, their neg_likelihood over the whole decode and their cluster counts.  An empty
    sequence returns no hypothesis.

    Speaker bounds (0 = none): an index tuple that would take its hypothesis past `max_speakers` clusters
    scores +inf; the returned hypothesis is the best-ranked final one with at least `min_speakers` clusters,
    or rank 0 when there is none."""
    self.rnn.eval()
    length = sequence.shape[0]
    tiled = torch.from_numpy(np.tile(sequence, (test_iteration, 1))).float().to(self.device)
    beam = [_Hypothesis()]
    for start in range(0, test_iteration * length, look_ahead):
      frames = tiled[start:start + look_ahead, :]
      depth = frames.shape[0]
      widest = max(len(h.means) for h in beam)
      scores = np.full([beam_size] + [widest + 1 + i for i in range(depth)], np.inf)
      for rank, hyp in enumerate(beam):
        table = self._score_table(hyp, frames, max_speakers)
        scores[rank] = np.pad(table, [(0, widest - len(hyp.means))] * depth, 'constant',
                              constant_values=np.inf)
      ranked = np.sort(scores, axis=None)
      ranked[ranked == np.inf] = 0
      finite = len(np.trim_zeros(ranked))
      order = np.argsort(scores, axis=None)
      survivors = []
      for rank in range(min(finite, beam_size)):
        index = np.unravel_index(order[rank], scores.shape)
        survivors.append(self._expand(beam[int(index[0])], frames, index[1:]))
      beam = survivors
    if n_best is not None:
      if length == 0:
        return [], [], []
      chosen = [beam[r] for r in nbest_ranks([len(h.means) for h in beam], min_speakers, n_best)]
      return ([[int(c) for c in h.trace[-length:]] for h in chosen], [float(h.score) for h in chosen],
              [len(h.means) for h in chosen])
    best = next((h for h in beam if len(h.means) >= min_speakers), beam[0])
    labels = [int(c) for c in best.trace[-length:]]
    return (labels, len(best.means)) if return_speakers else labels
