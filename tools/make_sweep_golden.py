"""Writes tests/golden/sweep_cases.npz: the REFERENCE's own decodes and losses under non-default (crp_alpha,
transition_bias) pairs -- what a decoding-parameter sweep (predict / score with decode_params) must reproduce.

TEST INFRASTRUCTURE ONLY, like oracle/make_golden.py (whose loaders it uses, and whose fixtures it leaves untouched):
it runs where the reference package is installed, never on the GPU box, and the tests read only the fixture it
writes.  The reference model is loaded from the golden weights with its crp_alpha / transition_bias set to each pair.

  toy_*     the toy model (model_toy100.npz) over toy_test utterances TOY_UTTS: predict_single labels per pair
            (toy_labels [C][frames], the utterances concatenated).  Pair 0 is the model's own, and its labels must
            reproduce toy_test.npz's.
  small_*   the D = 64 small model (model_small.npz) at look_ahead 2 over synthetic utterances (small_x, small_lengths,
            small_args = beam_size, look_ahead, test_iteration): per (pair c, utterance u) the reference's per-step
            trace as oracle/make_golden.py records it -- small_<c>_<u>_{labels,win,score,off,final_scores}.
  sc_*      per-frame losses of given labellings under non-default pairs (tools/make_score_golden.py's method):
            sc_<name>_{pair,labels,model,score,frames} and the rows (sc_<name>_toy_u >= 0: utterance of toy_test.npz,
            else sc_<name>_synth = [seed, n_frames, dim, n_spk, noise] for synth.synth_utt).
The tool asserts that, per model, every pair's labels differ from every other pair's on at least one utterance, so
that a config mix-up cannot pass a test that reads this file.

  python tools/make_sweep_golden.py [--jobs 4]"""
import argparse
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'oracle'))
sys.path.insert(0, os.path.join(REPO, 'tools'))
import make_golden as mg  # noqa: E402  (puts the reference package on sys.path)
import numpy as np  # noqa: E402
import torch  # noqa: E402
from make_score_golden import canonical, ref_score, synth_rows  # noqa: E402

TOY_UTTS = (0, 1, 2, 3, 4, 5)
TOY_PAIRS = ((1e-3, 0.5), (50.0, 0.2), (0.2, 0.9))        # after the model's own pair
SMALL_PAIRS = ((1e-3, 0.5), (30.0, 0.01), (0.2, 0.9))     # after the model's own pair
SMALL_UTTS = ((900, 24), (901, 24), (902, 24))            # synth seed, frames (dim 64, 3 speakers, noise 0.3)
SMALL_ARGS = dict(beam_size=5, look_ahead=2, test_iteration=2)


def with_pair(d, pair):
  d = dict(d)
  d['crp_alpha'], d['transition_bias'] = float(pair[0]), float(pair[1])
  return d


def own(d):
  return (float(d['crp_alpha']), float(d['transition_bias']))


def distinct(labels, what):
  """labels[c][u]: every pair's labels differ from every other pair's on some utterance."""
  for a in range(len(labels)):
    for b in range(a + 1, len(labels)):
      assert any(not np.array_equal(x, y) for x, y in zip(labels[a], labels[b])), '%s: pairs %d and %d agree' % (
          what, a, b)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--jobs', type=int, default=4)
  a = ap.parse_args()
  out = {}

  toy = np.load(os.path.join(mg.GOLD, 'toy_test.npz'))
  off = np.concatenate([[0], np.cumsum(toy['lengths'])])
  d = dict(np.load(os.path.join(mg.GOLD, 'model_toy100.npz')))
  pairs = [own(d)] + list(TOY_PAIRS)
  seqs = [toy['x'][off[u]:off[u + 1]].astype(np.float64) for u in TOY_UTTS]
  res = mg.pmap(mg._predict_worker, [(with_pair(d, p), s, {}) for p in pairs for s in seqs], a.jobs)  # pylint: disable=protected-access
  labels = [[res[c * len(seqs) + i][0] for i in range(len(seqs))] for c in range(len(pairs))]
  for i, u in enumerate(TOY_UTTS):
    assert np.array_equal(labels[0][i], toy['labels'][off[u]:off[u + 1]]), 'own pair does not reproduce toy_test'
  distinct(labels, 'toy')
  out['toy_pairs'] = np.array(pairs, np.float64)
  out['toy_utts'] = np.array(TOY_UTTS, np.int64)
  out['toy_labels'] = np.stack([np.concatenate(l) for l in labels])
  print('toy: %d pairs x %d utterances' % (len(pairs), len(seqs)), flush=True)

  d = dict(np.load(os.path.join(mg.GOLD, 'model_small.npz')))
  pairs = [own(d)] + list(SMALL_PAIRS)
  xs = [mg.synth.synth_utt(s, n_frames=n, dim=64, n_spk=3, noise=0.3)[0].astype(np.float32) for s, n in SMALL_UTTS]
  trs = mg.pmap(mg._trace_worker, [(with_pair(d, p), x, SMALL_ARGS) for p in pairs for x in xs], a.jobs)  # pylint: disable=protected-access
  distinct([[trs[c * len(xs) + i]['labels'] for i in range(len(xs))] for c in range(len(pairs))], 'small')
  out['small_pairs'] = np.array(pairs, np.float64)
  out['small_x'] = np.concatenate(xs)
  out['small_lengths'] = np.array([len(x) for x in xs], np.int64)
  out['small_args'] = np.array([SMALL_ARGS['beam_size'], SMALL_ARGS['look_ahead'], SMALL_ARGS['test_iteration']])
  for c in range(len(pairs)):
    for i in range(len(xs)):
      for key in ('labels', 'win', 'score', 'off', 'final_scores'):
        out['small_%d_%d_%s' % (c, i, key)] = trs[c * len(xs) + i][key]
  print('small: %d pairs x %d traced utterances' % (len(pairs), len(xs)), flush=True)

  torch.set_num_threads(4)
  names = []

  def add(name, fixture, pair, x, labs, toy_u=-1, synth=None):
    model = mg.model_from_dict(with_pair(dict(np.load(os.path.join(mg.GOLD, fixture))), pair))
    total, frames = ref_score(model, x, labs)
    names.append(name)
    out['sc_%s_pair' % name] = np.array(pair, np.float64)
    out['sc_%s_labels' % name] = labs
    out['sc_%s_model' % name] = np.array(fixture)
    out['sc_%s_toy_u' % name] = np.int64(toy_u)
    if synth is not None:
      out['sc_%s_synth' % name] = np.array(synth, np.float64)
    out['sc_%s_score' % name] = np.float64(total)
    out['sc_%s_frames' % name] = frames
    print('%-22s N=%4d score %.6g' % (name, len(labs), total), flush=True)

  u = 0
  x = toy['x'][off[u]:off[u + 1]]
  truth = canonical(toy['truth'][off[u]:off[u + 1]])
  for c, pair in enumerate(TOY_PAIRS):
    add('toy_truth_p%d' % (c + 1), 'model_toy100.npz', pair, x, truth, toy_u=u)
  args = (7401, 60, 64, 4, 0.08)
  lab = canonical(np.random.default_rng(7402).integers(0, 5, 60))
  for c, pair in enumerate(SMALL_PAIRS):
    add('s_random_p%d' % (c + 1), 'model_small.npz', pair, synth_rows(args), lab, synth=args)
  args = (7305, 4400, 64, 2, 0.08)  # more than 4096 speaker turns: past the default length of the log tables
  for c, pair in enumerate(SMALL_PAIRS[:2]):
    add('s_alternating_p%d' % (c + 1), 'model_small.npz', pair, synth_rows(args), np.arange(4400, dtype=np.int64) % 2,
        synth=args)
  out['sc_names'] = np.array(names)
  np.savez_compressed(os.path.join(mg.GOLD, 'sweep_cases.npz'), **out)


if __name__ == '__main__':
  main()
