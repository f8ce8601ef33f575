"""CPU oracle of predict() with speaker bounds -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

oracle/uis_oracle.py restates the reference's beam search; this module adds the two bounds on top of its
functions, with the semantics every implementation shares (include/uisrnn_b200.h, uis_predict_bounded):
  * max_speakers: an index tuple whose hypothesis would hold more than max_speakers clusters after
    _update_beam_state scores +inf; ranking, the flat-index tie-break and the min(#finite, B) cut are unchanged;
  * min_speakers: the returned hypothesis is the best-ranked final one with at least min_speakers clusters,
    else rank 0.
tests/golden/speaker_bounds_cases.npz was produced by the reference's own predict code with its _calculate_score
wrapped the same way (tools/make_speaker_bounds_golden.py); tests/test_speaker_bounds_cpu.py pins this module to it.
"""
import numpy as np

from helpers import uis_oracle as O


def clusters_after(k, cluster_seq):
  """len(mean_set) after _update_beam_state applies `cluster_seq` to a hypothesis with k clusters (valid tuples)."""
  for c in cluster_seq:
    if c == k:
      k += 1
  return k


def calculate_score(model, beam, chunk, max_speakers=0):
  table = O.calculate_score(model, beam, chunk)
  if max_speakers:
    for idx in np.argwhere(np.isfinite(table)):
      if clusters_after(len(beam.means), idx) > max_speakers:
        table[tuple(idx)] = np.inf
  return table


def predict_single(model, seq, beam_size=10, look_ahead=1, test_iteration=2, max_speakers=0, min_speakers=0,
                   record=None):
  """uis_oracle.predict_single with speaker bounds.  `record` also receives final_k (clusters per final rank),
  final_traces (labels of every final rank) and chosen (the rank the labels come from)."""
  n = seq.shape[0]
  tiled = np.tile(seq, (test_iteration, 1)).astype(O.F32)
  beams = [O.Beam()]
  win, sc, off, nfin = [], [], [0], []
  for t in range(0, test_iteration * n, look_ahead):
    chunk = tiled[t:t + look_ahead]
    la = chunk.shape[0]
    kmax = max(len(b.means) for b in beams)
    table = np.full([beam_size] + [kmax + 1 + i for i in range(la)], np.inf)
    for r, b in enumerate(beams):
      s = calculate_score(model, b, chunk, max_speakers)
      table[r] = np.pad(s, [(0, kmax - len(b.means))] * la, 'constant', constant_values=np.inf)
    ranked = np.sort(table, axis=None)
    ranked[ranked == np.inf] = 0
    ranked = np.trim_zeros(ranked)
    order = np.argsort(table, axis=None)
    new_beams = []
    for r in range(min(len(ranked), beam_size)):
      idx = np.unravel_index(order[r], table.shape)
      nb = O.update_beam_state(model, beams[int(idx[0])], chunk, idx[1:])
      new_beams.append(nb)
      win.append([int(v) for v in idx] + [-1] * (look_ahead - la))
      sc.append(float(nb.nl))
    off.append(len(win))
    nfin.append(len(ranked))
    beams = new_beams
  final_k = [len(b.means) for b in beams]
  chosen = next((r for r, k in enumerate(final_k) if k >= min_speakers), 0)
  if record is not None:
    record.update(
        win=np.array(win, dtype=np.int32).reshape(-1, 1 + look_ahead),
        score=np.array(sc, dtype=np.float64), off=np.array(off, dtype=np.int64),
        nfinite=np.array(nfin, dtype=np.int64),
        final_scores=np.array([float(b.nl) for b in beams]),
        final_k=np.array(final_k, dtype=np.int64),
        final_traces=np.array([b.trace[-n:] for b in beams], dtype=np.int64).reshape(len(beams), n),
        chosen=chosen)
  return [int(c) for c in beams[chosen].trace[-n:]]
