"""Float64 replay of a predict() trace -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A hypothesis's state depends only on its label history, and a trace (the debug taps of uis_predict: every step's
winners with their parent and index tuple, and their fp32 scores) gives that history for every hypothesis the search
kept.  Replaying the trace in float64 therefore yields, for every step and from the trace's own previous scores, what
the step should have produced: the increment of every candidate (parent x index tuple), which candidates should win,
and the states of the winners.  Each step is checked on its own terms however long the decode runs, and the check does
not depend on how exact ties were broken.

The replay keeps the quirks oracle/uis_oracle.py documents: the running mean (mu * (n - 1) + m) / n with n the visits
before this one; the log terms associated as mse - ((log p0 + log blocks) - log(tot + alpha)); weighted_mse's
first-column rule (d2[0] == 0 scores +inf); +inf for an invalid index; test_iteration tiling; a tail chunk shorter
than look_ahead; and the speaker bounds of include/uisrnn_b200.h (a candidate that takes its hypothesis past
max_speakers clusters is +inf; the labels come from the first final rank with at least min_speakers clusters, else
rank 0).  The GRU / MLP run in float64 on the fp32 weights; 1 / (2 sigma2) and the input rows are the fp32 values the
reference computes with.

Whether d2[0] is an exact fp32 zero cannot be decided from a float64 state: a candidate whose column-0 difference is
within ZERO_BAND is marked ambiguous (its +inf status is the kernel's to decide), except new-cluster candidates when
the kernel's own mean0 (uis_model_constants) is given, which decide it exactly."""
import contextlib
import types

import numpy as np

try:  # the replay's products are a few columns wide: a multi-threaded BLAS spends more time syncing than computing
  from threadpoolctl import threadpool_limits
except ImportError:  # pragma: no cover
  threadpool_limits = None

F32 = np.float32
# Bounds of the kernels' step checks (tests/test_gpu_step_replay.py, and the zero-padded shapes of
# tests/test_gpu_parity.py): about 10x the worst error of the unmodified kernels over test_gpu_step_replay.py on an H100
# 80GB HBM3 (700 W), given beside each, and never looser than the 1e-5 checks of test_gpu_parity.py.
INC_RTOL = 7e-7           # increment beyond one ulp of the score per sub-step, relative to |increment|: 6.9e-8
# best_mean / best_hidden rows, relative to the row's largest value: 3.3e-6 (the hidden state after a frame x1e3 once
# showed 7.2e-6); capped at the parity checks' 1e-5
STATE_TOL = 1e-5
# |mu[0] - x[0]| below this (times max(1, |x[0]|)) leaves the first-column rule undecided in float64
ZERO_BAND = 1e-5


def _f64(a):
  return np.asarray(a, dtype=np.float64)


class Model:
  """The weights of one model at its own (unpadded) shape, in float64."""

  def __init__(self, w):
    self.depth = int(w['depth'])
    self.w_ih = [_f64(np.asarray(w['weight_ih_l%d' % l], F32)) for l in range(self.depth)]
    self.w_hh = [_f64(np.asarray(w['weight_hh_l%d' % l], F32)) for l in range(self.depth)]
    self.b_ih = [_f64(np.asarray(w['bias_ih_l%d' % l], F32)) for l in range(self.depth)]
    self.b_hh = [_f64(np.asarray(w['bias_hh_l%d' % l], F32)) for l in range(self.depth)]
    self.w1, self.b1 = _f64(np.asarray(w['w1'], F32)), _f64(np.asarray(w['b1'], F32))
    self.w2, self.b2 = _f64(np.asarray(w['w2'], F32)), _f64(np.asarray(w['b2'], F32))
    self.H, self.D = self.w1.shape[0], self.w2.shape[0]
    self.h0 = _f64(np.asarray(w['h0'], F32)).reshape(self.depth, self.H)
    sigma2 = np.asarray(w['sigma2'], F32)
    self.w = _f64((F32(1.0) / (F32(2.0) * sigma2)).astype(F32))  # two fp32 tensor ops (uisrnn.py:414, 443)
    p0, alpha = float(w['transition_bias']), float(w['crp_alpha'])
    self.pen_last = np.log(1 - p0)
    self.log_p0, self.alpha = np.log(p0), alpha
    self.pen_new_head = np.log(p0) + np.log(alpha)
    m, h = self.core(np.zeros((1, self.D)), self.h0[None])
    self.mean0, self.hidden0 = m[0], h[0]

  def core(self, x, h):
    """CoreRNN on a batch of columns: x [n, D], h [n, depth, H] -> mean [n, D], hidden [n, depth, H].  numpy arrays,
    or float64 torch tensors (on any device: the weights follow them there)."""
    H = self.H
    w, xp = self._weights_like(x)
    inp, out = x, xp.empty_like(h)
    for l in range(self.depth):
      gi = inp @ w.w_ih[l].T + w.b_ih[l]
      gh = h[:, l] @ w.w_hh[l].T + w.b_hh[l]
      r = 1 / (1 + xp.exp(-(gi[:, :H] + gh[:, :H])))
      z = 1 / (1 + xp.exp(-(gi[:, H:2 * H] + gh[:, H:2 * H])))
      n = xp.tanh(gi[:, 2 * H:] + r * gh[:, 2 * H:])
      out[:, l] = (h[:, l] - n) * z + n
      inp = out[:, l]
    return (inp @ w.w1.T + w.b1).clip(min=0) @ w.w2.T + w.b2, out

  def _weights_like(self, x):
    if isinstance(x, np.ndarray):
      return self, np
    import torch
    cache = self.__dict__.setdefault('_on_device', {})
    if x.device not in cache:
      t = lambda a: torch.as_tensor(a, dtype=torch.float64, device=x.device)
      cache[x.device] = types.SimpleNamespace(
          w_ih=[t(a) for a in self.w_ih], w_hh=[t(a) for a in self.w_hh], b_ih=[t(a) for a in self.b_ih],
          b_hh=[t(a) for a in self.b_hh], w1=t(self.w1), b1=t(self.b1), w2=t(self.w2), b2=t(self.b2))
    return cache[x.device], torch


class Hyp:
  """A hypothesis: per cluster a node id (mean, hidden and visits live in the replay's node store), block counts,
  the last cluster and the kernel's fp32 score."""
  __slots__ = ('nodes', 'blocks', 'last', 'score')

  def __init__(self, nodes=(), blocks=(), last=-1, score=0.0):
    self.nodes, self.blocks, self.last, self.score = tuple(nodes), tuple(blocks), last, score

  @property
  def K(self):
    return len(self.nodes)


class Step:
  """What one beam step should have produced.
    t, la         first tiled frame of the chunk, sub-steps in it
    s_prev        [P] the kernel's scores of the parents (0 at the first step)
    inc           float64 table [P, K+1, K+2, ...] (K = the largest parent K): every candidate's increment, +inf for
                  an invalid index, a first-column zero, or a bound
    ambiguous     bool table of the same shape: +inf status undecided (first-column rule, see ZERO_BAND)
    tree          look_ahead >= 2: prefix tuple (parent, c1, .., cj) -> Hyp after j sub-steps (j < la)
    rows          the kernel's winner rows of this step (parent, c1, .., c_la)
    win_inc       [W] each winner's expected increment
    hyps          [W] the winners' states (Hyp; node data via Replay.node)"""
  __slots__ = ('t', 'la', 's_prev', 'inc', 'ambiguous', 'tree', 'rows', 'win_inc', 'hyps')


class Replay:
  """Replays one traced utterance; iterate over steps() to get a Step per beam step."""

  def __init__(self, weights, x, beam_size, look_ahead, test_iteration, win, score, off, max_speakers=0,
               min_speakers=0, mean0=None):
    self.m = weights if isinstance(weights, Model) else Model(weights)
    self.n = int(np.asarray(x).shape[0])
    self.x = np.tile(np.asarray(x, np.float64), (test_iteration, 1)).astype(F32).astype(np.float64)
    self.x32 = self.x.astype(F32)
    self.B, self.L = int(beam_size), int(look_ahead)
    self.win, self.score, self.off = np.asarray(win), np.asarray(score), np.asarray(off, np.int64)
    self.max_speakers, self.min_speakers = int(max_speakers or 0), int(min_speakers or 0)
    self.mean0_32 = None if mean0 is None else np.asarray(mean0, F32)
    self.store = {}   # node id -> (mean [D], hidden [depth, H], visits)
    self.next_id = 0
    self.hyps = [Hyp()]

  # ---- node store
  def node(self, nid):
    return self.store[nid]

  def _add(self, mean, hidden, visits):
    nid = self.next_id
    self.next_id += 1
    self.store[nid] = (mean, hidden, visits)
    return nid

  def _advance(self, keys, t):
    """New node ids for (source node id or -1 = a new cluster) visited at tiled frame t: one batched core per call,
    each distinct source evaluated once."""
    uniq = sorted(set(keys))
    if not uniq:
      return {}
    hs = np.stack([self.m.hidden0 if k < 0 else self.store[k][1] for k in uniq])
    mean, hid = self.m.core(np.repeat(self.x[t][None], len(uniq), 0), hs)
    out = {}
    for i, k in enumerate(uniq):
      if k < 0:
        out[k] = self._add(mean[i], hid[i], 1)
      else:
        mu, _, n = self.store[k]
        out[k] = self._add((mu * (n - 1) + mean[i]) / n, hid[i], n + 1)
    return out

  def _gc(self, live_hyps):
    live = {n for h in live_hyps for n in h.nodes}
    for k in [k for k in self.store if k not in live]:
      del self.store[k]

  # ---- one sub-step of scoring
  def _scores(self, hyps, t):
    """For every hyp, over c in 0..K (c == K: new cluster): (increment [K+1], ambiguous [K+1])."""
    x, x0 = self.x[t], self.x[t, 0]
    band = ZERO_BAND * max(1.0, abs(x0))
    ids = sorted({n for h in hyps for n in h.nodes})
    mse, d0 = {}, {}
    if ids:
      M = np.stack([self.store[k][0] for k in ids])
      v = ((M - x) ** 2) @ self.m.w
      for i, k in enumerate(ids):
        mse[k], d0[k] = v[i], M[i, 0] - x0
    mse0 = float(((self.m.mean0 - x) ** 2) @ self.m.w)
    if self.mean0_32 is not None:
      new_inf, new_amb = bool(self.mean0_32[0] == self.x32[t, 0]), False
    else:
      new_inf, new_amb = False, abs(self.m.mean0[0] - x0) <= band
    out = []
    for h in hyps:
      tot = sum(h.blocks)
      lt = np.log(tot + self.m.alpha)
      inc = np.empty(h.K + 1)
      amb = np.zeros(h.K + 1, bool)
      for c, k in enumerate(h.nodes):
        pen = self.m.pen_last if c == h.last else (self.m.log_p0 + np.log(h.blocks[c])) - lt
        inc[c] = mse[k] - pen
        amb[c] = abs(d0[k]) <= band
      inc[h.K] = np.inf if new_inf else mse0 - (self.m.pen_new_head - lt)
      amb[h.K] = new_amb
      if self.max_speakers and h.K + 1 > self.max_speakers:
        inc[h.K] = np.inf
        amb[h.K] = False
      out.append((inc, amb))
    return out

  @staticmethod
  def _moved(h, c, nid):
    """Hyp after visiting cluster c (c == K: new) with the cluster's new node id."""
    if c == h.K:
      return Hyp(h.nodes + (nid,), h.blocks + (1,), c)
    blocks = h.blocks if c == h.last else h.blocks[:c] + (h.blocks[c] + 1,) + h.blocks[c + 1:]
    return Hyp(h.nodes[:c] + (nid,) + h.nodes[c + 1:], blocks, c)

  def steps(self):
    T = self.x.shape[0]
    for s, t in enumerate(range(0, T, self.L)):
      la = min(self.L, T - t)
      st = Step()
      st.t, st.la = t, la
      st.s_prev = np.array([h.score for h in self.hyps], np.float64) if s else np.zeros(1)
      P = len(self.hyps)
      kmax = max(h.K for h in self.hyps)
      inc = np.full([P] + [kmax + 1 + i for i in range(la)], np.inf)
      amb = np.zeros(inc.shape, bool)
      # level by level over the tree of prefixes; a prefix's state is needed below the last level only
      level = [((b,), h, 0.0, False) for b, h in enumerate(self.hyps)]
      tree = {}
      for j in range(la):
        sc = self._scores([h for _, h, _, _ in level], t + j)
        if j == la - 1:
          for (pre, h, acc, a), (v, am) in zip(level, sc):
            inc[pre + (slice(0, h.K + 1),)] = acc + v
            amb[pre + (slice(0, h.K + 1),)] = a | am
          break
        children = []
        for (pre, h, acc, a), (v, am) in zip(level, sc):
          for c in range(h.K + 1):
            if np.isfinite(v[c]) or am[c]:
              children.append((pre + (c,), h, c, acc + v[c], a | am[c]))
        nids = self._advance([h.nodes[c] if c < h.K else -1 for _, h, c, _, _ in children], t + j)
        level = []
        for pre, h, c, acc, a in children:
          nh = self._moved(h, c, nids[h.nodes[c] if c < h.K else -1])
          tree[pre] = nh
          level.append((pre, nh, acc, a))
      # subtrees under an invalid / +inf prefix stay +inf (the table was filled with +inf)
      lo, hi = int(self.off[s]), int(self.off[s + 1])
      rows = self.win[lo:hi, :1 + la].astype(np.int64)
      st.inc, st.ambiguous, st.tree, st.rows = inc, amb, tree, rows
      st.win_inc = np.array([inc[tuple(r)] if self._valid(inc, r) else np.inf for r in rows])
      # winners' states: the prefix state of (parent, c1..c_{la-1}) advanced by the last sub-step
      last_src = []
      pre_states = []
      for r in rows:
        if not self._valid(inc, r):
          raise AssertionError('step %d: winner %s is not a valid index tuple' % (s, r.tolist()))
        h = self.hyps[r[0]] if la == 1 else tree.get(tuple(int(v) for v in r[:-1]))
        if h is None:
          raise AssertionError('step %d: winner %s extends a +inf or invalid prefix' % (s, r.tolist()))
        c = int(r[-1])
        if c > h.K:
          raise AssertionError('step %d: winner %s has an invalid cluster index' % (s, r.tolist()))
        pre_states.append((h, c))
        last_src.append(h.nodes[c] if c < h.K else -1)
      nids = self._advance(last_src, t + la - 1)
      new = []
      for (h, c), k, sc_ in zip(pre_states, last_src, self.score[lo:hi]):
        nh = self._moved(h, c, nids[k])
        nh.score = float(sc_)
        new.append(nh)
      st.hyps = new
      yield st
      self.hyps = new
      self._gc(new)

  @staticmethod
  def _valid(inc, r):
    return all(0 <= int(v) < n for v, n in zip(r, inc.shape))

  def chosen(self):
    """The final rank whose labels are returned (min_speakers rule)."""
    return next((r for r, h in enumerate(self.hyps) if h.K >= self.min_speakers), 0)


def backtrack(win, off, n, rank):
  """Labels of the last n tiled frames along the trace, from final rank `rank`."""
  labs = []
  r = rank
  for s in range(len(off) - 2, -1, -1):
    row = win[int(off[s]) + r]
    labs = [int(v) for v in row[1:] if v >= 0] + labs
    r = int(row[0])
    if len(labs) >= n:
      break
  return labs[len(labs) - n:] if n else []


def ulp32(v):
  return np.spacing(np.abs(np.asarray(v, np.float64)).astype(F32)).astype(np.float64)


def check(replay, inc_rtol, labels=None, final=None, state_tol=None, worst=None, visit=None):
  """Runs the replay and checks the trace step by step; raises AssertionError at the first violation.

    a. increment: |s[r] - s_prev[parent] - inc64| <= la * ulp32(s[r]) + inc_rtol * |inc64| (one fp32 accumulation
       per sub-step; the loss rounding and the kernel's own arithmetic go into inc_rtol)
    b. selection: #winners == min(#finite, B) (within the ambiguous candidates); the kernel's scores are
       non-decreasing; the winners are distinct; every winner's key s_prev + inc64 is <= every losing candidate's key
       and the ranked keys are non-decreasing, both up to the two candidates' step tolerances
    c. (final given: dict of best_mean, best_hidden, best_blocks, final_k, final_scores) the rank-0 state, each
       cluster's mean row and each (cluster, layer) hidden row within state_tol of its own largest value (floor 1e-2
       of the whole tensor's), blocks and K exact, final scores bit-equal to the last step's scores then +inf
    d. (labels given) the labels equal the back-track from the rank the min_speakers rule picks

  `worst` (a dict) receives the largest error per class: 'inc' (excess over the ulp allowance relative to |inc64|),
  'mean', 'hidden'.  `visit(step index, Step)` is called for every step after its checks.  Returns the labels of the
  back-track."""
  worst = {} if worst is None else worst
  with threadpool_limits(1, 'blas') if threadpool_limits else contextlib.nullcontext():
    return _check(replay, inc_rtol, labels, final, state_tol, worst, visit)


def _check(replay, inc_rtol, labels, final, state_tol, worst, visit):
  bump = lambda k, v: worst.__setitem__(k, max(worst.get(k, 0.0), float(v)))
  nsteps = 0
  for s, st in enumerate(replay.steps()):
    nsteps += 1
    rows, sc = st.rows, np.asarray(replay.score[replay.off[s]:replay.off[s + 1]], np.float64)
    where = 'step %d (frame %d)' % (s, st.t)
    # b. count
    finite = np.isfinite(st.inc) & ~st.ambiguous
    nf, na = int(finite.sum()), int((st.ambiguous).sum())
    W = len(rows)
    assert min(nf, replay.B) <= W <= min(nf + na, replay.B), \
        '%s: %d winners, %d finite candidates (+%d undecided), beam %d' % (where, W, nf, na, replay.B)
    assert W > 0
    # a. increments
    par = rows[:, 0]
    allow = st.la * ulp32(sc)
    assert np.all(np.isfinite(sc)), '%s: a winner has a non-finite score' % where
    amb_w = np.array([st.ambiguous[tuple(r)] for r in rows])
    assert np.all(np.isfinite(st.win_inc) | amb_w), '%s: a winner is +inf in the replay' % where
    ok = np.isfinite(st.win_inc)
    err = np.abs(sc - st.s_prev[par] - st.win_inc)
    excess = np.where(ok, (err - allow) / np.abs(st.win_inc), 0.0)
    bump('inc', excess.max())
    bad = ok & (err > allow + inc_rtol * np.abs(st.win_inc))
    assert not bad.any(), '%s rank %d: score %.9g, parent %.9g + increment %.12g (error %.3g, allowed %.3g)' % (
        where, int(np.argmax(bad)), sc[bad][0], st.s_prev[par][bad][0], st.win_inc[bad][0], err[bad][0],
        (allow + inc_rtol * np.abs(st.win_inc))[bad][0])
    # b. order and selection
    assert np.all(np.diff(sc) >= 0), '%s: kernel scores not ranked' % where
    flat = np.ravel_multi_index(tuple(rows.T), st.inc.shape)
    assert len(set(flat.tolist())) == W, '%s: a candidate won twice' % where
    key = st.s_prev.reshape([-1] + [1] * st.la) + st.inc
    tol = st.la * ulp32(np.where(np.isfinite(key), key, 0)) + inc_rtol * np.abs(np.where(np.isfinite(st.inc), st.inc, 0))
    kw, tw = key.ravel()[flat], tol.ravel()[flat]
    kw, tw = kw[ok], tw[ok]
    assert np.all(kw[:-1] - tw[:-1] <= kw[1:] + tw[1:]), '%s: ranks out of order beyond tolerance' % where
    lose = finite.ravel().copy()
    lose[flat] = False
    if lose.any() and kw.size:
      lo_up = (key.ravel() + tol.ravel())[lose]
      assert np.max(kw - tw) <= np.min(lo_up), \
          '%s: winner key %.9g above a losing candidate key %.9g' % (where, np.max(kw - tw), np.min(lo_up))
    if visit:
      visit(s, st)
  last = replay.hyps
  labs = backtrack(replay.win, replay.off, replay.n, replay.chosen()) if nsteps else []
  if labels is not None:
    assert list(labels) == labs, 'labels differ from the back-track of the trace'
  if final is not None and nsteps:
    best = last[0]
    assert int(final['final_k']) == best.K
    assert np.array_equal(np.asarray(final['best_blocks']).reshape(-1), np.array(best.blocks))
    means = np.stack([replay.node(k)[0] for k in best.nodes])
    hids = np.stack([replay.node(k)[1] for k in best.nodes])
    gm = np.asarray(final['best_mean'], np.float64).reshape(means.shape)
    gh = np.asarray(final['best_hidden'], np.float64).reshape(hids.shape)
    em = np.max(np.abs(gm - means), axis=1) / np.maximum(np.max(np.abs(means), axis=1), 1e-2 * np.max(np.abs(means)))
    eh = np.max(np.abs(gh - hids), axis=2) / np.maximum(np.max(np.abs(hids), axis=2), 1e-2 * np.max(np.abs(hids)))
    bump('mean', em.max())
    bump('hidden', eh.max())
    assert em.max() <= state_tol, 'best_mean row %d: error %.3g of its scale' % (int(np.argmax(em)), em.max())
    assert eh.max() <= state_tol, 'best_hidden: error %.3g of its scale' % eh.max()
    fs = np.asarray(final['final_scores'], np.float64)
    lastsc = np.asarray(replay.score[replay.off[-2]:replay.off[-1]], np.float64)
    assert np.array_equal(fs[:len(lastsc)], lastsc) and np.all(np.isinf(fs[len(lastsc):]))
  return labs


def frame_allowance(inc, gauss, inc_rtol=INC_RTOL):
  """How far a kernel's fp32 per-frame increment may lie from the float64 one: one fp32 ulp of the increment (its final
  rounding) plus inc_rtol times the frame's Gaussian term.  Beyond that rounding the only error of an increment is the
  fp32 weighted mse (the log terms are float64), so the bound scales with the Gaussian term, not with the increment,
  which cancellation against the log terms can make small."""
  with np.errstate(invalid='ignore'):
    return ulp32(inc) + inc_rtol * np.asarray(gauss, np.float64)


def frame_share(got, inc, gauss, inc_rtol=INC_RTOL):
  """|got - inc| / frame_allowance per frame (<= 1 within it; 0 where equal, +inf included; +inf where exactly one of
  the two is +inf)."""
  got, inc = np.asarray(got, np.float64), np.asarray(inc, np.float64)
  with np.errstate(invalid='ignore', divide='ignore'):
    share = np.abs(got - inc) / frame_allowance(inc, gauss, inc_rtol)
  return np.where(got == inc, 0.0, np.where(np.isnan(share), np.inf, share))


class PathScores:
  """What path_score returns, per path: `score`, the float64 neg_likelihood; and the two parts of the allowance an
  fp32 accumulation of the same path may differ by, as check() bounds each step: `ulps`, one fp32 ulp of the running
  score per sub-step, and `mass`, the sum of |increment| (the part INC_RTOL scales).  Absent paths are nan.

  With path_score(per_frame=True), also per path (lists in the same order, None for an absent path): `frame_inc`, the
  float64 increment of every frame, and `frame_gauss`, its Gaussian term (the weighted mse; +inf under the
  first-column rule)."""

  def __init__(self, score, ulps, mass, frame_inc=None, frame_gauss=None):
    self.score, self.ulps, self.mass = score, ulps, mass
    self.frame_inc, self.frame_gauss = frame_inc, frame_gauss

  def frame_share(self, got, inc_rtol=INC_RTOL):
    """frame_share of every path's fp32 per-frame increments in `got` (a list in path order): a list of arrays."""
    return [frame_share(g, i, s, inc_rtol) for g, i, s in zip(got, self.frame_inc, self.frame_gauss)]

  def allowance(self, inc_rtol=INC_RTOL):
    return self.ulps + inc_rtol * self.mass

  def share(self, got, inc_rtol=INC_RTOL):
    """|got - score| / allowance: how much of its allowance each fp32 score in `got` uses (<= 1 within it; +inf for
    a path the float64 search scores +inf, 0 for an empty one)."""
    err = np.abs(np.asarray(got, np.float64) - self.score)
    with np.errstate(invalid='ignore', divide='ignore'):
      return np.where(err == 0, 0.0, err / self.allowance(inc_rtol))


def path_score(model, xs, labels, mean0=None, device='cpu', max_slots=1 << 17, per_frame=False):
  """Float64 rescoring of given label paths: the neg_likelihood the search assigns to a hypothesis whose cluster at
  frame t is labels[t], summed over the frames with the score terms of Replay (running-mean off-by-one, log-term
  association, first-column rule; `mean0`, the kernel's fp32 mean0, decides that rule exactly for new clusters).

    xs      list of [N_u, D] inputs, already tiled (np.tile(x, (test_iteration, 1))) when the path covers the tiling
    labels  list of int [R_u, N_u]: R_u paths over utterance u; a row of -1 is an absent rank (nan scores)

  Returns a PathScores of arrays [sum R_u] in (utterance, row) order; per_frame=True adds every path's float64
  per-frame increments and Gaussian terms (PathScores.frame_inc / frame_gauss).  A path is its labels only at
  look_ahead 1 or any look_ahead (the sub-steps of a tree step add the same per-frame increments), but only over the
  whole tiled decode: predict() returns the last tiled copy, which at test_iteration > 1 leaves the earlier copies' labels, and so
  every cluster's state, undetermined.  Rescore those from the back-track of a trace instead.

  Batched in torch float64 on `device`: one GRU product per frame over every path of every utterance, each cluster
  state evaluated once however many paths share it (a cluster's state depends only on the frames it holds so far, so
  paths that agree on those share a node).  Utterances are taken in groups of at most `max_slots` cluster slots."""
  import torch
  m = model if isinstance(model, Model) else Model(model)
  dev = torch.device(device)
  f64 = dict(dtype=torch.float64, device=dev)
  rows = [np.atleast_2d(np.asarray(lab, np.int64)) for lab in labels]
  assert all(r.shape[1] == len(x) for x, r in zip(xs, rows)), 'labels and inputs of different lengths'
  first = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
  out = [np.full(int(first[-1]), np.nan) for _ in range(3)]
  frames = [[None] * int(first[-1]) for _ in range(2)] if per_frame else None  # increments, Gaussian terms
  w = torch.as_tensor(m.w, **f64)
  mean0_64 = torch.as_tensor(m.mean0, **f64)
  hidden0 = torch.as_tensor(m.hidden0, **f64)
  new0 = None if mean0 is None else float(np.asarray(mean0, F32)[0])
  inf = torch.tensor(np.inf, dtype=torch.float32, device=dev)
  # groups of utterances: a path of K clusters holds K slots
  groups, cur, slots = [], [], 0
  for u, r in enumerate(rows):
    k = int(np.maximum(r.max(axis=1, initial=-1), -1).sum() + len(r)) if r.size else 0
    if cur and slots + k > max_slots:
      groups.append(cur)
      cur, slots = [], 0
    cur.append(u)
    slots += k
  groups.append(cur)
  with torch.no_grad():
    for us in groups:
      paths = [(u, j) for u in us for j in range(len(rows[u])) if rows[u].shape[1] == 0 or rows[u][j, 0] >= 0]
      if not paths:
        continue
      n_p = np.array([rows[u].shape[1] for u, _ in paths], np.int64)
      lab = np.full((len(paths), max(1, int(n_p.max()))), -1, np.int64)
      for p, (u, j) in enumerate(paths):
        lab[p, :n_p[p]] = rows[u][j]
      if (lab[np.arange(lab.shape[1]) < n_p[:, None]] < 0).any():
        raise ValueError('a path has a -1 label inside its frames')
      kp = lab.max(axis=1) + 1
      base = np.concatenate([[0], np.cumsum(kp)[:-1]]).astype(np.int64)
      S = int(kp.sum())
      xg = [np.asarray(xs[u], np.float64).astype(F32) for u in us]
      xoff = np.concatenate([[0], np.cumsum([len(x) for x in xg])]).astype(np.int64)
      pos = {u: i for i, u in enumerate(us)}
      X = torch.as_tensor(np.concatenate(xg).reshape(-1, m.D), device=dev)
      utt = torch.as_tensor(np.array([pos[u] for u, _ in paths], np.int64), device=dev)
      xrow = torch.as_tensor(xoff[[pos[u] for u, _ in paths]], device=dev)
      lab_t, n_t, base_t = (torch.as_tensor(a, device=dev) for a in (lab, n_p, base))
      mean = torch.zeros((S, m.D), **f64)
      hid = torch.zeros((S, m.depth, m.H), **f64)
      visits = torch.zeros(S, **f64)
      blocks = torch.zeros(S, **f64)
      nid = torch.full((S,), -1, dtype=torch.int64, device=dev)
      P = len(paths)
      K = torch.zeros(P, dtype=torch.int64, device=dev)
      last = torch.full((P,), -1, dtype=torch.int64, device=dev)
      tot = torch.zeros(P, **f64)
      score, ulps, mass = torch.zeros(P, **f64), torch.zeros(P, **f64), torch.zeros(P, **f64)
      if per_frame:
        f_inc, f_gauss = torch.zeros((P, lab.shape[1]), **f64), torch.zeros((P, lab.shape[1]), **f64)
      next_id = 0
      for t in range(int(n_p.max())):
        live = torch.nonzero(n_t > t).squeeze(1)
        c = lab_t[live, t]
        Kl = K[live]
        if bool((c > Kl).any()):
          raise ValueError('frame %d: a label skips a cluster (labels open clusters in order 0, 1, ..)' % t)
        new = c == Kl
        slot = base_t[live] + c
        x32 = X[xrow[live] + t]
        x = x32.double()
        # score terms (Replay._scores)
        mu = torch.where(new[:, None], mean0_64[None], mean[slot])
        d = mu - x
        mse = (d * d) @ w
        if new0 is None:
          zero = d[:, 0] == 0
        else:
          zero = torch.where(new, x32[:, 0] == new0, d[:, 0] == 0)
        mse = torch.where(zero, inf.double(), mse)
        lt = torch.log(tot[live] + m.alpha)
        pen = torch.where(new, m.pen_new_head - lt,
                          torch.where(c == last[live], torch.full_like(lt, m.pen_last),
                                      (m.log_p0 + torch.log(blocks[slot])) - lt))
        inc = mse - pen
        if per_frame:
          f_inc[live, t] = inc
          f_gauss[live, t] = mse
        s = score[live] + inc
        score[live] = s
        a = s.abs().float()
        ulps[live] += (torch.nextafter(a, inf) - a).double()
        mass[live] += inc.abs()
        # hypothesis bookkeeping (Replay._moved)
        turn = new | (c != last[live])
        blocks[slot] = blocks[slot] + turn.double()
        tot[live] = tot[live] + turn.double()
        K[live] = Kl + new.long()
        last[live] = c
        # advance the visited cluster: one core per distinct source state (Replay._advance)
        key = torch.where(new, -1 - utt[live], nid[slot])
        uniq, inv = torch.unique(key, return_inverse=True)
        rep = torch.empty(len(uniq), dtype=torch.int64, device=dev).scatter_(
            0, inv, torch.arange(len(inv), device=dev))
        rs, rn = slot[rep], new[rep]
        mo, ho = m.core(x[rep], torch.where(rn[:, None, None], hidden0[None], hid[rs]))
        v = visits[rs]
        mo = torch.where(rn[:, None], mo, (mean[rs] * (v - 1)[:, None] + mo) / v.clamp(min=1)[:, None])
        mean[slot] = mo[inv]
        hid[slot] = ho[inv]
        visits[slot] = torch.where(new, torch.ones_like(v[inv]), visits[slot] + 1)
        nid[slot] = next_id + inv
        next_id += len(uniq)
      idx = np.array([first[u] + j for u, j in paths], np.int64)
      for o, v in zip(out, (score, ulps, mass)):
        o[idx] = v.cpu().numpy()
      if per_frame:
        for o, v in zip(frames, (f_inc.cpu().numpy(), f_gauss.cpu().numpy())):
          for p, i in enumerate(idx):
            o[i] = v[p, :n_p[p]]
  return PathScores(*out, *(frames or ()))
