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
  s_alternating                two speakers alternating every frame over 4400 frames: more than 4096 speaker turns,
                               past the default length of the kernels' log tables (model_small.npz)
  s_3000_clusters              one utterance of 4200 frames in 3000 clusters, mostly singletons and pairs
                               (model_small.npz)

Per case: <name>_labels, <name>_model, <name>_score (the total) and <name>_frames, the reference's own per-frame
loss (float32 [N]: what _update_beam_state adds to neg_likelihood at each frame, fl32(f64(mse32) - pen)).  The rows
are utterance <name>_toy_u of toy_test.npz, or <name>_x, or -- to keep the fixture small for the two long cases --
synth.synth_utt(seed, n_frames, dim, n_spk, noise=noise) of <name>_synth = [seed, n_frames, dim, n_spk, noise],
cast to float32 as here.  Regenerating must reproduce every earlier case's labels and total bit for bit (asserted
against the fixture being replaced).

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
  """(neg_likelihood, float32 per-frame losses) of the reference's _update_beam_state driven along `labels`.  Each
  frame's call starts from neg_likelihood 0, so that it returns the frame's loss itself; the running sum then adds it
  the way _update_beam_state's `neg_likelihood += loss` does."""
  model.rnn_model.eval()
  rows = torch.from_numpy(np.asarray(x, np.float32))
  state = mg.ref_mod.BeamState()
  frames = np.zeros(len(labels), np.float32)
  with torch.no_grad():
    for t, c in enumerate(labels):
      total = state.neg_likelihood
      state.neg_likelihood = 0
      state = model._update_beam_state(state, rows[t:t + 1], (int(c),))  # pylint: disable=protected-access
      loss = state.neg_likelihood
      assert np.asarray(loss).dtype == np.float32
      frames[t] = loss
      state.neg_likelihood = total + loss
  return float(state.neg_likelihood), frames


def synth_rows(args):
  seed, n, dim, n_spk, noise = args
  return mg.synth.synth_utt(int(seed), n_frames=int(n), dim=int(dim), n_spk=int(n_spk), noise=float(noise))[0]


def random_labels(rng, n, k, singletons):
  lab = rng.integers(0, k, n)
  lab[rng.choice(n, singletons, replace=False)] = k + np.arange(singletons)  # clusters of one frame each
  return canonical(lab)


def main():
  torch.set_num_threads(4)
  out, names = {}, []

  path = os.path.join(mg.GOLD, 'score_cases.npz')
  old = dict(np.load(path)) if os.path.exists(path) else {}

  def add(name, fixture, x, labels, model, toy_u=-1, synth=None):
    total, frames = ref_score(model, x, labels)
    names.append(name)
    if synth is not None:
      out[name + '_synth'] = np.array(synth, np.float64)
    elif toy_u < 0:
      out[name + '_x'] = np.asarray(x, np.float32)
    out[name + '_toy_u'] = np.int64(toy_u)  # >= 0: the rows are utterance toy_u of toy_test.npz
    out[name + '_labels'] = labels
    out[name + '_model'] = np.array(fixture)
    out[name + '_score'] = np.float64(total)
    out[name + '_frames'] = frames
    for key in ('_x', '_labels', '_score'):
      if name + key in old:
        assert np.array_equal(old[name + key], out[name + key]), 'regenerated %s%s differs' % (name, key)
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
  args = (7305, 4400, 64, 2, 0.08)
  add('s_alternating', 'model_small.npz', synth_rows(args), np.arange(4400, dtype=np.int64) % 2, small, synth=args)
  args = (7306, 4200, 64, 4, 0.08)
  lab = np.random.default_rng(7307).permutation(np.concatenate([np.arange(1800), 1800 + np.arange(2400) // 2]))
  add('s_3000_clusters', 'model_small.npz', synth_rows(args), canonical(lab), small, synth=args)
  assert out['s_3000_clusters_labels'].max() + 1 == 3000
  out['names'] = np.array(names)
  np.savez_compressed(path, **out)


if __name__ == '__main__':
  main()
