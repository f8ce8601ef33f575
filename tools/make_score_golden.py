"""Writes tests/golden/score_cases.npz: the REFERENCE's own neg_likelihood of given labellings.

TEST INFRASTRUCTURE ONLY, like oracle/make_golden.py (whose loaders it uses): it runs where the reference package
is installed, never on the GPU box, and the tests read only the fixture it writes.  Every score is the
`neg_likelihood` the reference's `_update_beam_state` (uisrnn/uisrnn.py:388-453) accumulates when it is driven along
the labelling frame by frame from an empty BeamState -- the quantity UISRNN.score() returns.

Cases (labels stored canonical: 0, 1, 2, ... in order of first appearance):
  toy_truth_<u>, toy_ref_<u>   the toy test utterances with their true labels and the reference's decoded labels
                               (model_toy100.npz)
  s_singletons, s_one_speaker, s_many   random labellings with many one-frame clusters, a one-speaker utterance and
                               one with 40 clusters (model_small.npz)
  d2_random                    a random labelling with the depth-2 model (model_small_d2.npz)

  python tools/make_score_golden.py"""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'oracle'))
import make_golden as mg  # noqa: E402  (puts the reference package on sys.path)
import numpy as np  # noqa: E402
import torch  # noqa: E402


def canonical(ids):
  seen = {}
  return np.array([seen.setdefault(int(v), len(seen)) for v in ids], np.int64)


def ref_score(model, x, labels):
  """neg_likelihood of the reference's _update_beam_state driven along `labels`."""
  model.rnn_model.eval()
  rows = torch.from_numpy(np.asarray(x, np.float32))
  state = mg.ref_mod.BeamState()
  with torch.no_grad():
    for t, c in enumerate(labels):
      state = model._update_beam_state(state, rows[t:t + 1], (int(c),))  # pylint: disable=protected-access
  return float(state.neg_likelihood)


def random_labels(rng, n, k, singletons):
  lab = rng.integers(0, k, n)
  lab[rng.choice(n, singletons, replace=False)] = k + np.arange(singletons)  # clusters of one frame each
  return canonical(lab)


def main():
  torch.set_num_threads(4)
  out, names = {}, []

  def add(name, fixture, x, labels, model, toy_u=-1):
    total = ref_score(model, x, labels)
    names.append(name)
    if toy_u < 0:
      out[name + '_x'] = np.asarray(x, np.float32)
    out[name + '_toy_u'] = np.int64(toy_u)  # >= 0: the rows are utterance toy_u of toy_test.npz
    out[name + '_labels'] = labels
    out[name + '_model'] = np.array(fixture)
    out[name + '_score'] = np.float64(total)
    print('%-16s N=%4d K=%3d score %.6g' % (name, len(labels), labels.max() + 1 if len(labels) else 0, total), flush=True)

  toy = np.load(os.path.join(mg.GOLD, 'toy_test.npz'))
  model = mg.model_from_dict(dict(np.load(os.path.join(mg.GOLD, 'model_toy100.npz'))))
  off = np.concatenate([[0], np.cumsum(toy['lengths'])])
  for u in range(int(toy['n_utt'])):
    x = toy['x'][off[u]:off[u + 1]]
    add('toy_truth_%d' % u, 'model_toy100.npz', x, canonical(toy['truth'][off[u]:off[u + 1]]), model, u)
    add('toy_ref_%d' % u, 'model_toy100.npz', x, canonical(toy['labels'][off[u]:off[u + 1]]), model, u)

  rng = np.random.default_rng(7301)
  small = mg.model_from_dict(dict(np.load(os.path.join(mg.GOLD, 'model_small.npz'))))
  x = mg.synth.synth_utt(7302, n_frames=60, dim=64, n_spk=4, noise=0.08)[0]
  add('s_singletons', 'model_small.npz', x, random_labels(rng, 60, 3, 12), small)
  add('s_one_speaker', 'model_small.npz', x, np.zeros(60, np.int64), small)
  x = mg.synth.synth_utt(7303, n_frames=90, dim=64, n_spk=5, noise=0.08)[0]
  add('s_many', 'model_small.npz', x, random_labels(rng, 90, 20, 20), small)
  assert out['s_many_labels'].max() + 1 > 32
  d2 = mg.model_from_dict(dict(np.load(os.path.join(mg.GOLD, 'model_small_d2.npz'))))
  x = mg.synth.synth_utt(7304, n_frames=50, dim=64, n_spk=4, noise=0.08)[0]
  add('d2_random', 'model_small_d2.npz', x, random_labels(rng, 50, 4, 5), d2)
  out['names'] = np.array(names)
  np.savez_compressed(os.path.join(mg.GOLD, 'score_cases.npz'), **out)


if __name__ == '__main__':
  main()
