"""Data-parallel fit() steps pinned per element to the float64 oracle of a fit() iteration (tests/fit_oracle.py).

A data-parallel iteration is uis_trainer_step(mode 2) on each rank's columns (gradients left un-normalised: the
backward pass takes a row count of 1), uis_trainer_comm_export, an all-reduce(sum) and uis_trainer_comm_apply
(division by the global row count, loss1 / loss2 / the sigma2 gradient from the summed per-dimension statistics,
then the regulariser, clip and Adam).  Without dropout it is, in exact arithmetic, the full-batch iteration, so the
oracle is fit_oracle.losses_and_grads on the full batch; with dropout each rank masks its own shard layout under its
own seed (fit_oracle.shard_dropout_scales).

One GPU stands in for W ranks: each rank is its own NativeTrainer; a rank with columns steps in mode 2 and exports,
a rank without columns exports nothing and contributes a zero buffer (as UISRNN._fit_native does), the sum is a torch
fp32 add, and every rank applies it.  After every apply each rank's gradients (normalised, regulariser included,
unclipped) and losses are checked per element against the oracle with the local scales and bounds of
test_gpu_fit_fp64.py (GRAD_TOL, LOSS_RTOL, FLOOR, OPT_TOL, E2E_*: imported, not restated), and the ranks' parameters,
gradients and losses must be bit-identical.

Unlike the stand-ins that compare parameters after an Adam step (whose first update lr * g / (|g| + eps) hides any
positive scale of g), these checks see the scale of every gradient: a shard that still divides by its local row
count, an h0 gradient left un-normalised or dropout masks of the wrong iteration fail here.

The cases reach the trainer's paths in data-parallel mode: the persistent recurrence (H = 128, 512, 1024) and the
per-step launches (H = 100), 64x64 GEMM tiles (D = 65), depth 1..3, shards that cross 32-column groups and shards of
>= 256 columns (the sliced column sum), per-rank row counts that differ, ranks that hold no column of a mini-batch
(whose first trainer call is then comm_apply), inter-layer dropout, the optimiser and the corpus route (step_corpus
after set_corpus / set_corpus_device)."""
import numpy as np
import pytest

import fit_oracle
import test_gpu_fit_fp64 as fp64
from test_gpu_fit_fp64 import (E2E_LOSS_RTOL, E2E_PARAM_MAX, E2E_PARAM_P99, HP, OPT_TOL, check_grads, check_losses,
                               record, trainer_for)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method='thread')]


@pytest.fixture(scope='module', autouse=True)
def worst_per_class():
  """check_grads / check_losses record into test_gpu_fit_fp64.WORST: collect this file's figures apart and print
  them at the end (pytest -s)."""
  saved, fp64.WORST = fp64.WORST, {}
  yield fp64.WORST
  worst = fp64.WORST
  fp64.WORST = saved
  print('\ndata-parallel fit vs float64, worst error per class:')
  for cls in sorted(worst):
    print('  %-14s %.2e  %s' % (cls, worst[cls][0], worst[cls][1]))


def layout_lengths(name):
  rng = np.random.default_rng(sum(map(ord, name)))
  if name == 'b520':   # 520 columns: over two ranks each shard is >= 256 columns wide (9 groups, sliced column sum)
    return [12] + sorted(rng.integers(2, 13, 519).tolist(), reverse=True)
  if name == 'b5':     # five columns: over eight ranks, ranks 5..7 hold none
    return [14, 11, 9, 5, 2]
  return fp64.layout_lengths(name)


def batch(shape, layout, it=0):
  D, H, _ = shape
  return fit_oracle.make_batch(layout_lengths(layout), D, seed=H + 100 * it, zeros=layout == 'zeros')


def dp_iteration(trainers, B, shard_step):
  """One data-parallel iteration of ranks `trainers` over a B-column mini-batch.  shard_step(trainer, columns) runs
  the mode-2 step of a rank on its columns.  The buffer of a rank with columns starts as NaN, so that a slot
  comm_export leaves unwritten poisons the sum.  Returns each rank's losses of the iteration."""
  import torch
  from uisrnn_b200.uisrnn import shard_columns
  world = len(trainers)
  total = None
  for r, tr in enumerate(trainers):
    mine = shard_columns(B, r, world)
    if len(mine):
      buf = torch.full((tr.comm_size(),), float('nan'), device='cuda')
      shard_step(tr, mine)
      tr.comm_export(buf.data_ptr())
    else:
      buf = torch.zeros(tr.comm_size(), device='cuda')
    total = buf if total is None else total + buf
  for tr in trainers:
    tr.comm_apply(total.data_ptr())
  return [tuple(float(v) for v in tr.losses(1)[0]) for tr in trainers]


def host_shards(x, lengths):
  """shard_step of a host batch: the rank's columns, cut to the length of its first one."""
  def step(tr, mine):
    ll = lengths[mine]
    tr.step_shard(np.ascontiguousarray(x[:ll[0], mine]), ll)
  return step


def check_replicas(trainers, grads0):
  """Every rank holds the same parameters, gradients and losses as rank 0, bit for bit."""
  p0, l0 = trainers[0].parameters(), trainers[0].losses(1)
  for r, tr in enumerate(trainers[1:], 1):
    p, g = tr.parameters(), tr.gradients()
    for k in p0:
      assert np.array_equal(p[k], p0[k]), ('parameters', r, k)
      assert np.array_equal(g[k], grads0[k]), ('gradients', r, k)
    assert np.array_equal(tr.losses(1), l0), ('losses', r)


def check_ranks(trainers, losses, want_losses, want, depth, what):
  for r, tr in enumerate(trainers):
    check_losses(losses[r], want_losses, what=what + (r,))
    check_grads(tr.gradients(), want, depth, what=what + (r,))
  check_replicas(trainers, trainers[0].gradients())


def run_dp(shape, layout, world, iterations=1, p=0.0):
  """`iterations` data-parallel iterations of `world` ranks (per-rank dropout seeds when p > 0), each against the
  oracle of the full batch from the parameters the ranks held before it."""
  D, H, depth = shape
  params = fit_oracle.random_params(D, H, depth, seed=1000 * depth + H + D)
  seeds = [0x5DEECE66D + 7919 * r for r in range(world)]
  trainers = [trainer_for(params, HP, dropout=p, dropout_seed=seeds[r]) for r in range(world)]
  try:
    for it in range(iterations):
      x, lengths = batch(shape, layout, it)
      before = trainers[0].parameters()
      losses = dp_iteration(trainers, len(lengths), host_shards(x, lengths))
      scales = fit_oracle.shard_dropout_scales(seeds, it, depth, lengths, H, p, world) if p > 0 else None
      want_losses, want = fit_oracle.losses_and_grads(before, x, lengths, HP, scales=scales, device='cuda')
      check_ranks(trainers, losses, want_losses, want, depth, (shape, layout, world, it))
  finally:
    for tr in trainers:
      tr.close()


SHAPES = [(64, 128, 1), (256, 512, 2), (40, 100, 3), (65, 129, 1), (512, 1024, 1)]
CASES = ([(s, 'b33', 2) for s in SHAPES] + [(s, 'b33', 3) for s in SHAPES[:4]] +
         [(s, lay, w) for s in [(64, 128, 1), (256, 512, 2), (40, 100, 3), (65, 129, 1)]
          for lay, w in (('b64', 2), ('extreme', 2), ('extreme', 3), ('zeros', 2), ('zeros', 3), ('b520', 2))])


def _id(case):
  (D, H, depth), layout, world = case
  return 'D{}-H{}-depth{}-{}-world{}'.format(D, H, depth, layout, world)


@pytest.mark.parametrize('case', CASES, ids=_id)
def test_data_parallel_step_matches_fp64(case):
  run_dp(*case)


IDLE_CASES = [((64, 128, 1), 'min', 2), ((64, 128, 1), 'b5', 8), ((40, 100, 3), 'b5', 8)]


@pytest.mark.parametrize('case', IDLE_CASES, ids=_id)
def test_ranks_without_columns_match_fp64(case):
  """Mini-batches narrower than the world: the ranks past the batch width export nothing, add zeros and apply
  the sum -- their first trainer call is comm_apply -- and two iterations later still hold the model every other
  rank holds."""
  run_dp(*case, iterations=2)


@pytest.mark.parametrize('shape', [(64, 128, 3), (40, 100, 3)], ids=['persistent-depth3', 'per_step-depth3'])
def test_inter_layer_dropout_matches_fp64(shape):
  """p = 0.3, three ranks with their own seeds, two iterations: each rank masks its own shard layout with the
  iteration number it shares with the others."""
  run_dp(shape, 'b33', 3, iterations=2, p=0.3)


@pytest.mark.parametrize('name', ['default', 'clip', 'sigma2_clamp'])
def test_optimizer_step_matches_fp64_adam(name):
  """Six full data-parallel steps over three ranks (the optimiser cases of test_gpu_fit_fp64.py): every rank's
  parameters after apply are the oracle's clip + Adam + clamp of the step's parameters and gradients."""
  overrides, special = fp64.OPT_CASES[name]
  hp = dict(HP, **overrides)
  shape = (64, 128, 2)
  D = shape[0]
  params, _, _ = fp64.case_inputs(shape, 'b33', seed=5)
  if special == 'sigma2':
    params['sigma2'][:D // 4] = 5e-3
  world = 3
  trainers = [trainer_for(params, hp) for _ in range(world)]
  adam = fit_oracle.FitAdam(params, hp)
  lr = hp['learning_rate']
  try:
    for step in range(6):
      x, lengths = fit_oracle.make_batch(fp64.layout_lengths('b33'), D, seed=300 + step)
      before = trainers[0].parameters()
      dp_iteration(trainers, len(lengths), host_shards(x, lengths))
      grads = trainers[0].gradients()
      check_replicas(trainers, grads)
      want = adam.step(grads, params=before)
      if name == 'clip':
        assert adam.clip_coef < 1e-3, adam.clip_coef
      for r, tr in enumerate(trainers):
        got = tr.parameters()
        for k in want:
          w32 = np.float32(want[k])
          err = np.abs(got[k].astype(np.float64) - want[k]) - np.spacing(np.abs(w32)).astype(np.float64)
          record('adam', float(err.max()) / lr, (name, step, r, k))
          assert float(err.max()) <= OPT_TOL * lr, (name, step, r, k, float(err.max()) / lr)
        if special == 'sigma2' and step == 0:
          assert np.all(got['sigma2'][:D // 4] == np.float32(1e-6))
  finally:
    for tr in trainers:
      tr.close()


def test_short_trajectory_matches_fp64():
  """Five full data-parallel steps at the config-4 shape over three ranks, the oracle running its own full-batch
  iterations and Adam from the same start: the losses of every step and the parameters after the last."""
  shape = (256, 512, 2)
  D = shape[0]
  params, _, _ = fp64.case_inputs(shape, 'b33', seed=9)
  trainers = [trainer_for(params, HP) for _ in range(3)]
  adam = fit_oracle.FitAdam(params, HP)
  ref = {k: np.asarray(v, np.float64) for k, v in params.items()}
  try:
    for step in range(5):
      x, lengths = fit_oracle.make_batch(fp64.layout_lengths('b33'), D, seed=500 + step)
      losses = dp_iteration(trainers, len(lengths), host_shards(x, lengths))
      want_losses, grads = fit_oracle.losses_and_grads(ref, x, lengths, HP, device='cuda')
      for r in range(3):
        check_losses(losses[r], want_losses, rtol=E2E_LOSS_RTOL, what=('step', step, r), cls='e2e_loss')
      ref = adam.step(grads)
    check_replicas(trainers, trainers[0].gradients())
    got = trainers[0].parameters()
  finally:
    for tr in trainers:
      tr.close()
  for k in ref:
    d = np.abs(got[k] - ref[k]) / HP['learning_rate']
    record('e2e_param_max', float(d.max()), k)
    record('e2e_param_p99', float(np.percentile(d, 99)), k)
    assert d.max() <= E2E_PARAM_MAX and np.percentile(d, 99) <= E2E_PARAM_P99, (k, d.max(), np.percentile(d, 99))


def _corpus(D, seed=17):
  """A float64 training set [600, D] and 70 sub-sequences of 1..20 row indices (as utils.resize_indices gives)."""
  rng = np.random.default_rng(seed)
  rows = rng.normal(0, 0.3, (600, D)) + rng.normal(0, 1, (1, D))
  index_lists = [rng.choice(600, n, replace=False).astype(np.int32) for n in rng.integers(1, 21, 70)]
  return rows, index_lists


def _host_batch(rows, index_lists, chosen):
  """The batch uis_trainer_step_corpus gathers, built on the host: row 0 zero, column b = rows of sub-sequence
  chosen[b] rounded to float32, zero padding."""
  lengths = np.array([len(index_lists[c]) + 1 for c in chosen], np.int32)
  x = np.zeros((int(lengths[0]), len(chosen), rows.shape[1]), np.float32)
  for b, c in enumerate(chosen):
    x[1:lengths[b], b] = rows[index_lists[c]]
  return x, lengths


@pytest.mark.parametrize('source', ['set_corpus', 'set_corpus_device-bfloat16'])
def test_corpus_route_matches_fp64(source):
  """step_corpus(chosen[mine], mode=2) on three ranks whose training set is on the device (copied from float64
  rows, or bfloat16 rows read in place), against the oracle of the batch built on the host from the same rows.
  That host batch is first shown to be the batch the trainer gathers: a mode-1 step on it gives the gradients of a
  mode-1 step_corpus bit for bit.  sigma2's is the exception: it is formed from the loss kernel's atomic
  per-dimension sums, whose order varies from run to run, so it is compared within 1e-5 of its largest element."""
  import torch
  shape = (64, 128, 1)
  D, H, depth = shape
  rows, index_lists = _corpus(D)
  tensors = None
  if source != 'set_corpus':
    t = torch.from_numpy(rows).cuda().bfloat16()
    tensors = [t[:250], t[250:]]
    rows = t.double().cpu().numpy()   # the exact values the trainer reads

  def load(tr):
    if tensors is None:
      tr.set_corpus(rows, index_lists)
    else:
      tr.set_corpus_device(tensors, index_lists)

  params = fit_oracle.random_params(D, H, depth, seed=31)
  rng = np.random.default_rng(5)
  lens = np.array([len(ix) for ix in index_lists])
  draws = []
  for _ in range(2):
    ids = rng.choice(len(index_lists), 40, replace=False)
    draws.append(ids[np.argsort(-lens[ids], kind='stable')].astype(np.int32))

  gathered, host = trainer_for(params, HP), trainer_for(params, HP)
  try:
    load(gathered)
    gathered.step_corpus(draws[0], mode=1)
    x, lengths = _host_batch(rows, index_lists, draws[0])
    host.step(x, lengths, grads_only=True)
    g, h = gathered.gradients(), host.gradients()
    for k in h:
      if k == 'sigma2':   # its terms cancel: the atomic order shows against the largest element, not each one
        assert np.max(np.abs(g[k] - h[k])) <= 1e-5 * np.max(np.abs(h[k])), k
      else:
        assert np.array_equal(g[k], h[k]), k
  finally:
    gathered.close()
    host.close()

  trainers = [trainer_for(params, HP) for _ in range(3)]
  try:
    for tr in trainers:
      load(tr)
    for it, chosen in enumerate(draws):
      x, lengths = _host_batch(rows, index_lists, chosen)
      before = trainers[0].parameters()
      losses = dp_iteration(trainers, len(chosen), lambda tr, mine: tr.step_corpus(chosen[mine], mode=2))
      want_losses, want = fit_oracle.losses_and_grads(before, x, lengths, HP, device='cuda')
      check_ranks(trainers, losses, want_losses, want, depth, (source, it))
  finally:
    for tr in trainers:
      tr.close()
