"""ctypes binding of libuisrnn_b200.so (C ABI in include/uisrnn_b200.h).

This is the only place the Python host code touches the native library.  There is no CPU
fallback here: if the shared library is missing or a call fails, an exception is raised.
"""
import ctypes as C
import os
import threading

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# UISRNN_B200_LIB: developer switch for A/B runs of differently tuned builds (tools/); default = the in-tree build
LIB_PATH = os.environ.get('UISRNN_B200_LIB') or os.path.join(_HERE, 'libuisrnn_b200.so')

UIS_OK = 0
UIS_ERR_INVALID = -1
UIS_ERR_UNSUPPORTED = -2
UIS_ERR_CUDA = -3
UIS_ERR_OVERFLOW = -4
UIS_ERR_NOMEM = -5
UIS_ERR_CAPACITY = -6
UIS_ABI_VERSION = 7  # include/uisrnn_b200.h


class NativeError(RuntimeError):
  def __init__(self, code, message):
    super().__init__('libuisrnn_b200: {} (code {})'.format(message, code))
    self.code = code


class PredictOpts(C.Structure):
  _fields_ = [('beam_size', C.c_int32), ('look_ahead', C.c_int32), ('test_iteration', C.c_int32),
              ('kcap', C.c_int32), ('n_ctas', C.c_int32), ('lanes', C.c_int32), ('cluster', C.c_int32),
              ('engine', C.c_int32)]


class DebugTaps(C.Structure):
  _fields_ = [('trace_utt', C.c_int32), ('trace_capacity', C.c_int32),
              ('step_winners', C.POINTER(C.c_int32)), ('step_scores', C.POINTER(C.c_float)),
              ('step_offsets', C.POINTER(C.c_int64)), ('final_scores', C.POINTER(C.c_float)),
              ('final_k', C.POINTER(C.c_int32)), ('best_mean', C.POINTER(C.c_float)),
              ('best_hidden', C.POINTER(C.c_float)), ('best_blocks', C.POINTER(C.c_int32))]


class NBestOut(C.Structure):
  _fields_ = [('labels_out', C.POINTER(C.c_void_p)), ('labels_dev', C.c_void_p), ('scores', C.POINTER(C.c_float)),
              ('speakers', C.POINTER(C.c_int32)), ('count', C.POINTER(C.c_int32))]


class DecodeParams(C.Structure):
  _fields_ = [('count', C.c_int32), ('crp_alpha', C.POINTER(C.c_double)), ('transition_bias', C.POINTER(C.c_double))]


class Stats(C.Structure):
  _fields_ = [('utterances', C.c_int64), ('frames', C.c_int64), ('beam_steps', C.c_int64),
              ('gru_columns', C.c_int64), ('weight_passes', C.c_int64), ('candidates', C.c_int64),
              ('kernel_launches', C.c_int64), ('ctas', C.c_int32), ('max_k', C.c_int32),
              ('prepass_ms', C.c_float), ('beam_ms', C.c_float), ('lanes', C.c_int32), ('cluster', C.c_int32), ('engine', C.c_int32),
              ('tc_columns', C.c_int32), ('phase_cycles', C.c_int64 * 10), ('tc_cycles', C.c_int64 * 4),
              ('h2d_ms', C.c_float), ('pipeline_ms', C.c_float), ('host_ms', C.c_float), ('chunks', C.c_int32),
              ('groups', C.c_int32), ('staged', C.c_int32)]

  def as_dict(self):
    out = {}
    for k, t in self._fields_:
      v = getattr(self, k)
      out[k] = float(v) if t is C.c_float else (list(v) if hasattr(v, '__len__') else int(v))
    return out


# Every symbol include/uisrnn_b200.h declares (tests check the .so exports all of them).
EXPORTS = ('uis_version', 'uis_last_error', 'uis_model_create', 'uis_model_destroy',
           'uis_model_constants', 'uis_predict', 'uis_predict_device', 'uis_predict_bounded',
           'uis_predict_device_bounded', 'uis_predict_nbest', 'uis_predict_device_nbest',
           'uis_score', 'uis_score_device', 'uis_predict_sweep', 'uis_predict_device_sweep', 'uis_score_sweep',
           'uis_score_device_sweep', 'uis_score_device_ids', 'uis_predict_workspace_bytes', 'uis_get_stats', 'uis_trainer_create',
           'uis_trainer_destroy', 'uis_trainer_step', 'uis_trainer_get', 'uis_trainer_losses',
           'uis_trainer_comm_size', 'uis_trainer_comm_export', 'uis_trainer_comm_apply',
           'uis_trainer_set_corpus', 'uis_trainer_step_corpus', 'uis_trainer_set_corpus_device')

# uis_dtype: the element types uis_trainer_set_corpus_device reads
UIS_DTYPE_F32, UIS_DTYPE_F16, UIS_DTYPE_BF16, UIS_DTYPE_F64 = 0, 1, 2, 3


class TrainHParams(C.Structure):
  _fields_ = [('learning_rate', C.c_float), ('sigma_alpha', C.c_float), ('sigma_beta', C.c_float),
              ('regularization_weight', C.c_float), ('grad_max_norm', C.c_float),
              ('train_sigma2', C.c_int32), ('rnn_depth', C.c_int32), ('rnn_dropout', C.c_float),
              ('dropout_seed', C.c_int64)]


def param_order(depth=1):
  """Names of the 4 * depth + 6 training tensors in the order uis_trainer_create takes them."""
  names = []
  for layer in range(depth):
    names += ['gru.{}_l{}'.format(kind, layer) for kind in ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh')]
  return tuple(names + ['linear_mean1.weight', 'linear_mean1.bias', 'linear_mean2.weight', 'linear_mean2.bias',
                        'rnn_init_hidden', 'sigma2'])


PARAM_ORDER = param_order(1)


def dropout_keep_mask(seed, iteration, layer, count, p):
  """The keep decisions of uis_train.cu's dropout_kernel for elements 0..count-1 (bool array): the same 32-bit
  hash, restated in numpy -- used by the tests to rebuild the masks of a training iteration."""
  seed = np.uint32((int(seed) ^ (int(seed) >> 32)) & 0xffffffff)
  with np.errstate(over='ignore'):
    i = np.arange(count, dtype=np.uint32)
    h = seed ^ (np.uint32(iteration) * np.uint32(0x9E3779B1)) ^ (np.uint32(layer) * np.uint32(0x85EBCA77)) ^ \
        (i * np.uint32(0xC2B2AE3D))
    h ^= h >> np.uint32(16); h *= np.uint32(0x7FEB352D); h ^= h >> np.uint32(15); h *= np.uint32(0x846CA68B)
    h ^= h >> np.uint32(16)
  u = (h >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
  return u >= np.float32(p)

_lib = None


def load_library():
  """Loads the shared library (once).  Raises if it has not been built."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    raise NativeError(UIS_ERR_INVALID,
                      'native library not built: {} is missing (run `python -c "import '
                      '__graft_entry__ as g; g.build()"`)'.format(LIB_PATH))
  lib = C.CDLL(LIB_PATH)
  fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int32)
  lib.uis_version.restype = C.c_int
  # the structs below are laid out for exactly one ABI version: a stale binary (the .so is built out of band and
  # git-ignored) must not be driven with mismatching layouts
  if lib.uis_version() != UIS_ABI_VERSION:
    raise NativeError(UIS_ERR_INVALID, '{} reports ABI version {}, this binding needs {}: rebuild it (python -c '
                      '"import __graft_entry__ as g; g.build()")'.format(LIB_PATH, lib.uis_version(), UIS_ABI_VERSION))
  if not os.environ.get('UISRNN_B200_LIB'):
    try:
      from . import build as _build
      if _build.is_stale():
        import warnings
        warnings.warn('libuisrnn_b200.so is older than its sources (uisrnn_b200/csrc); rebuild with '
                      '__graft_entry__.build()', RuntimeWarning)
    except OSError:
      pass
  lib.uis_last_error.restype = C.c_char_p
  lib.uis_model_create.restype = C.c_int
  lib.uis_model_create.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_int] + \
      [C.c_void_p] * 10 + [C.c_double, C.c_double]
  lib.uis_model_destroy.restype = C.c_int
  lib.uis_model_destroy.argtypes = [C.c_void_p]
  lib.uis_model_constants.restype = C.c_int
  lib.uis_model_constants.argtypes = [C.c_void_p, fp, fp]
  lib.uis_predict.restype = C.c_int
  lib.uis_predict.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int,
                              C.POINTER(PredictOpts), C.POINTER(C.c_void_p),
                              C.POINTER(DebugTaps), C.c_void_p]
  lib.uis_predict_device.restype = C.c_int
  lib.uis_predict_device.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int,
                                     C.POINTER(PredictOpts), C.c_void_p, C.POINTER(DebugTaps),
                                     C.c_void_p]
  lib.uis_predict_bounded.restype = C.c_int
  lib.uis_predict_bounded.argtypes = lib.uis_predict.argtypes + [ip, ip, ip]
  lib.uis_predict_device_bounded.restype = C.c_int
  lib.uis_predict_device_bounded.argtypes = lib.uis_predict_device.argtypes + [ip, ip, C.c_void_p]
  lib.uis_predict_nbest.restype = C.c_int
  lib.uis_predict_nbest.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int,
                                    C.POINTER(PredictOpts), C.POINTER(DebugTaps), C.c_void_p, ip, ip, C.c_int32,
                                    C.POINTER(NBestOut)]
  lib.uis_predict_device_nbest.restype = C.c_int
  lib.uis_predict_device_nbest.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int,
                                           C.POINTER(PredictOpts), C.POINTER(DebugTaps), C.c_void_p, ip, ip,
                                           C.c_int32, C.POINTER(NBestOut)]
  lib.uis_score.restype = C.c_int
  lib.uis_score.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int, C.POINTER(C.c_void_p),
                            fp, C.POINTER(C.c_void_p), C.c_void_p]
  lib.uis_score_device.restype = C.c_int
  lib.uis_score_device.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p]
  lib.uis_predict_sweep.restype = C.c_int
  lib.uis_predict_sweep.argtypes = lib.uis_predict_nbest.argtypes + [C.POINTER(DecodeParams)]
  lib.uis_predict_device_sweep.restype = C.c_int
  lib.uis_predict_device_sweep.argtypes = lib.uis_predict_device_nbest.argtypes + [C.POINTER(DecodeParams)]
  lib.uis_score_sweep.restype = C.c_int
  lib.uis_score_sweep.argtypes = lib.uis_score.argtypes + [C.POINTER(DecodeParams)]
  lib.uis_score_device_sweep.restype = C.c_int
  lib.uis_score_device_sweep.argtypes = lib.uis_score_device.argtypes + [C.POINTER(DecodeParams)]
  lib.uis_score_device_ids.restype = C.c_int
  lib.uis_score_device_ids.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(DecodeParams)]
  lib.uis_predict_workspace_bytes.restype = C.c_size_t
  lib.uis_predict_workspace_bytes.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.c_int,
                                              C.POINTER(PredictOpts)]
  lib.uis_get_stats.restype = C.c_int
  lib.uis_get_stats.argtypes = [C.c_void_p, C.POINTER(Stats)]
  lib.uis_trainer_create.restype = C.c_int
  lib.uis_trainer_create.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int,
                                     C.POINTER(C.c_void_p), C.POINTER(TrainHParams)]
  lib.uis_trainer_destroy.restype = C.c_int
  lib.uis_trainer_destroy.argtypes = [C.c_void_p]
  lib.uis_trainer_step.restype = C.c_int
  lib.uis_trainer_step.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.c_int, C.c_int, C.c_int,
                                   fp, C.c_void_p]
  lib.uis_trainer_get.restype = C.c_int
  lib.uis_trainer_get.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
  lib.uis_trainer_losses.restype = C.c_int
  lib.uis_trainer_losses.argtypes = [C.c_void_p, C.c_int, fp]
  lib.uis_trainer_set_corpus.restype = C.c_int
  lib.uis_trainer_set_corpus.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32]
  lib.uis_trainer_step_corpus.restype = C.c_int
  lib.uis_trainer_step_corpus.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, fp, C.c_void_p]
  lib.uis_trainer_set_corpus_device.restype = C.c_int
  lib.uis_trainer_set_corpus_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_int64,
                                                C.c_void_p, C.c_int32, C.c_void_p]
  lib.uis_trainer_comm_size.restype = C.c_int64
  lib.uis_trainer_comm_size.argtypes = [C.c_void_p]
  lib.uis_trainer_comm_export.restype = C.c_int
  lib.uis_trainer_comm_export.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
  lib.uis_trainer_comm_apply.restype = C.c_int
  lib.uis_trainer_comm_apply.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
  _lib = lib
  return lib


def _check(lib, rc):
  if rc != 0:
    raise NativeError(rc, lib.uis_last_error().decode('utf-8', 'replace'))


def _f32(a):
  return np.ascontiguousarray(a, dtype=np.float32)


def speaker_bounds(n, max_speakers=None, min_speakers=None):
  """(max, min) as int32 arrays of length n, or None for an absent bound.  An int applies to every utterance, a
  sequence gives one value per utterance; 0 means no bound.  Raises ValueError for a value that is not an integer (floats
  and bools included, scalar or not), a negative value, a wrong length, or min > max where both are set."""
  out = []
  for name, v in (('max_speakers', max_speakers), ('min_speakers', min_speakers)):
    if v is None:
      out.append(None)
      continue
    a = np.asarray(v)
    if a.ndim == 0:
      a = np.full(n, v, a.dtype)
    elif a.ndim != 1 or len(a) != n:
      raise ValueError('{} needs one value per utterance ({}), got shape {}'.format(name, n, a.shape))
    if (a.size or np.ndim(v) == 0) and not np.issubdtype(a.dtype, np.integer):  # (an empty list has a float dtype)
      raise ValueError('{} must be integers, got {}'.format(name, a.dtype))
    if (a < 0).any():
      raise ValueError('{} must be >= 0 (0 = no bound)'.format(name))
    out.append(np.ascontiguousarray(a, dtype=np.int32))
  mx, mn = out
  if mx is not None and mn is not None and ((mx > 0) & (mn > mx)).any():
    raise ValueError('min_speakers must not exceed max_speakers')
  return mx, mn


def check_n_best(n_best, beam_size):
  """Raises ValueError unless n_best is an int in [1, beam_size]."""
  if isinstance(n_best, (bool, np.bool_)) or not isinstance(n_best, (int, np.integer)):
    raise ValueError('n_best must be an int, got {!r}'.format(n_best))
  if not 1 <= n_best <= beam_size:
    raise ValueError('n_best must be in [1, beam_size={}], got {}'.format(beam_size, n_best))
  return int(n_best)


def decode_params(pairs):
  """(crp_alpha, transition_bias) float64 arrays of a sweep: a non-empty sequence of pairs, crp_alpha finite and > 0,
  transition_bias finite and in (0, 1).  Raises ValueError naming the first bad pair."""
  if isinstance(pairs, (str, bytes)) or not hasattr(pairs, '__len__') or len(pairs) == 0:
    raise ValueError('decode_params must be a non-empty sequence of (crp_alpha, transition_bias) pairs')
  alpha, p0 = np.empty(len(pairs), np.float64), np.empty(len(pairs), np.float64)
  for c, pair in enumerate(pairs):
    try:
      a, b = pair
      alpha[c], p0[c] = float(a), float(b)
    except (TypeError, ValueError):
      raise ValueError('decode_params pair {}: {!r} is not a (crp_alpha, transition_bias) pair of floats'.format(
          c, pair)) from None
    if isinstance(a, (bool, np.bool_)) or isinstance(b, (bool, np.bool_)):
      raise ValueError('decode_params pair {}: {!r} is not a (crp_alpha, transition_bias) pair of floats'.format(c, pair))
    if not (np.isfinite(alpha[c]) and alpha[c] > 0):
      raise ValueError('decode_params pair {}: crp_alpha={!r} (need finite and > 0)'.format(c, a))
    if not (np.isfinite(p0[c]) and 0 < p0[c] < 1):
      raise ValueError('decode_params pair {}: transition_bias={!r} (need finite and in (0, 1))'.format(c, b))
  return alpha, p0


def _decode_struct(pairs):
  """(DecodeParams, keep-alive arrays, count) of a validated sweep."""
  alpha, p0 = decode_params(pairs)
  dp = C.POINTER(C.c_double)
  return DecodeParams(len(alpha), alpha.ctypes.data_as(dp), p0.ctypes.data_as(dp)), (alpha, p0), len(alpha)


def _trim_taps(bufs, trace_utt):
  """Debug taps cut to what the call wrote: the traced job's step rows and its best hypothesis' clusters."""
  nrows = int(bufs['off'][-1]) if len(bufs['off']) else 0
  bufs['win'] = bufs['win'][:nrows]
  bufs['score'] = bufs['score'][:nrows]
  k = int(bufs['final_k'][trace_utt]) if trace_utt >= 0 else 0
  for key in ('best_mean', 'best_hidden', 'best_blocks'):
    bufs[key] = bufs[key][:k]
  return bufs


class NativeModel:
  """Owns a `uis_model*`.  Weights are numpy arrays in PyTorch state_dict layout."""

  def __init__(self, weights, device=0):
    lib = load_library()
    self._lib = lib
    self._h = C.c_void_p()
    w = weights
    depth = int(w.get('depth', 1))
    self.H = int(np.asarray(w['w1']).shape[0])
    self.D = int(np.asarray(w['w2']).shape[0])
    self.device = device
    self.depth = depth
    self.lock = threading.Lock()  # callers sharing this handle between threads serialise on it
    H, D = self.H, self.D
    layers = range(depth)
    for l in layers:  # PyTorch nn.GRU layouts: layer 0 sees the observation, layer l >= 1 sees layer l-1
      if tuple(np.asarray(w['weight_ih_l%d' % l]).shape) != (3 * H, D if l == 0 else H) or \
         tuple(np.asarray(w['weight_hh_l%d' % l]).shape) != (3 * H, H):
        raise ValueError('GRU weight shapes of layer %d do not match hidden=%d dim=%d' % (l, H, D))
    cat = lambda key: _f32(np.concatenate([np.asarray(w['%s_l%d' % (key, l)], np.float32).reshape(-1) for l in layers]))
    arrs = [cat('weight_ih'), cat('weight_hh'), cat('bias_ih'), cat('bias_hh'),
            _f32(w['w1']), _f32(w['b1']), _f32(w['w2']), _f32(w['b2']),
            _f32(np.asarray(w['h0']).reshape(-1)), _f32(w['sigma2'])]
    expect = [None, None, (depth * 3 * H,), (depth * 3 * H,), (H, H), (H,), (D, H), (D,), (depth * H,), (D,)]
    for a, e in zip(arrs, expect):
      if e is not None and tuple(a.shape) != e:
        raise ValueError('weight shape {} != expected {}'.format(a.shape, e))
    ptrs = [a.ctypes.data_as(C.c_void_p) for a in arrs]
    self.crp_alpha, self.transition_bias = float(w['crp_alpha']), float(w['transition_bias'])
    _check(lib, lib.uis_model_create(C.byref(self._h), device, self.D, self.H, depth, *ptrs,
                                     self.transition_bias, self.crp_alpha))
    # the model's own pair as a one-pair sweep: the call every entry point without decode_params makes
    self._own = (np.array([self.crp_alpha]), np.array([self.transition_bias]))
    dp = C.POINTER(C.c_double)
    self._own_dp = DecodeParams(1, self._own[0].ctypes.data_as(dp), self._own[1].ctypes.data_as(dp))

  def close(self):
    if getattr(self, '_h', None) is not None and self._h:
      self._lib.uis_model_destroy(self._h)
      self._h = C.c_void_p()

  def __del__(self):
    try:
      self.close()
    except Exception:  # pylint: disable=broad-except
      pass

  def constants(self):
    mean0 = np.empty(self.D, np.float32)
    hidden0 = np.empty((self.depth, self.H), np.float32)
    fp = C.POINTER(C.c_float)
    _check(self._lib, self._lib.uis_model_constants(self._h, mean0.ctypes.data_as(fp),
                                                    hidden0.ctypes.data_as(fp)))
    return mean0, hidden0

  @staticmethod
  def _opts(beam_size, look_ahead, test_iteration, kcap, n_ctas, lanes=0, cluster=0, engine=0):
    return PredictOpts(int(beam_size), int(look_ahead), int(test_iteration), int(kcap), int(n_ctas),
                       int(lanes), int(cluster), int(engine))

  def _taps(self, trace_utt, n_utt, lengths, beam_size, look_ahead, test_iteration, kcap):
    """Allocates host buffers for the debug taps; returns (struct, dict of arrays)."""
    kcap = kcap or (32 if look_ahead == 1 else 16)
    steps = -(-int(lengths[trace_utt]) * test_iteration // look_ahead) if trace_utt >= 0 else 0
    cap = max(1, steps * beam_size)
    bufs = {
        'win': np.full((cap, 1 + look_ahead), -1, np.int32),
        'score': np.zeros(cap, np.float32),
        'off': np.zeros(steps + 1, np.int64),
        'final_scores': np.zeros((n_utt, beam_size), np.float32),
        'final_k': np.zeros(n_utt, np.int32),
        'best_mean': np.zeros((kcap, self.D), np.float32),
        'best_hidden': np.zeros((kcap, self.depth, self.H), np.float32),
        'best_blocks': np.zeros(kcap, np.int32),
    }
    fp, ip, lp = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_int64)
    t = DebugTaps(int(trace_utt), int(cap), bufs['win'].ctypes.data_as(ip),
                  bufs['score'].ctypes.data_as(fp), bufs['off'].ctypes.data_as(lp),
                  bufs['final_scores'].ctypes.data_as(fp), bufs['final_k'].ctypes.data_as(ip),
                  bufs['best_mean'].ctypes.data_as(fp), bufs['best_hidden'].ctypes.data_as(fp),
                  bufs['best_blocks'].ctypes.data_as(ip))
    return t, bufs

  def _rows(self, seqs):
    """(arrays, lengths, offsets) of host utterances: each as a C-contiguous float64 [N_u, D] array (the caller's own
    when it already is one), their int64 lengths (one 0 entry for an empty list) and frame offsets [U + 1]."""
    n = len(seqs)
    keep = [s if (type(s) is np.ndarray and s.dtype == np.float64 and s.flags.c_contiguous)
            else np.ascontiguousarray(s, dtype=np.float64) for s in seqs]
    for s in keep:
      if s.ndim != 2 or s.shape[1] != self.D:
        raise ValueError('utterance shape {} does not match D={}'.format(s.shape, self.D))
    lens = np.fromiter((s.shape[0] for s in keep), dtype=np.int64, count=n) if n else np.zeros(1, np.int64)
    offs = np.zeros(n + 1, np.int64)
    np.cumsum(lens[:n], out=offs[1:])
    return keep, lens, offs

  def _sweep(self, decode_params):
    """(DecodeParams, keep-alive arrays, count) of a sweep; None is the model's own pair."""
    return (self._own_dp, None, 1) if decode_params is None else _decode_struct(decode_params)

  def predict(self, seqs, beam_size=10, look_ahead=1, test_iteration=2, kcap=0, n_ctas=0,
              trace_utt=None, stream=0, lanes=0, cluster=0, engine=0, max_speakers=None, min_speakers=None,
              return_speakers=False, n_best=None):
    """seqs: list of C-contiguous float64 [N_u, D] arrays (host).  Returns a list of int32
    label arrays (and a dict of debug arrays when trace_utt is not None).

    n_best=k (1 <= k <= beam_size): returns (labels, scores, speakers, count) instead, where labels[u] is int32
    [k][N_u] (row 0 = the labels of the same call without n_best), scores float32 [U][k] (neg_likelihood, +inf where
    absent), speakers int32 [U][k] and count int32 [U]; return_speakers is ignored.

    max_speakers / min_speakers: an int for every utterance or one value per utterance, 0 = no bound
    (uis_predict_bounded in include/uisrnn_b200.h).  return_speakers=True appends an int32 array with the
    cluster count of every returned hypothesis to the result.

    This is predict_sweep() under the model's own pair, reshaped: hypothesis 0 at n_best 1 is what uis_predict_bounded
    returns."""
    out = self.predict_sweep(seqs, None, beam_size, look_ahead, test_iteration, kcap, n_ctas, trace_utt, stream, lanes,
                             cluster, engine, max_speakers, min_speakers, n_best)
    (labels, scores, speakers, count), bufs = out if trace_utt is not None else (out, None)
    if n_best is not None:
      out = ([lab[0] for lab in labels], scores[0], speakers[0], count[0])
    elif return_speakers:
      out = ([lab[0, 0] for lab in labels], speakers[0, :, 0])
    else:
      out = [lab[0, 0] for lab in labels]
    return (out, bufs) if bufs is not None else out

  def predict_device(self, x_ptr, frame_offsets, labels_ptr, beam_size=10, look_ahead=1,
                     test_iteration=2, kcap=0, n_ctas=0, stream=0, lanes=0, cluster=0, engine=0,
                     max_speakers=None, min_speakers=None, speakers_ptr=0, n_best=None, scores_ptr=0,
                     nbest_speakers_ptr=0, count_ptr=0):
    """Device-resident variant: x_ptr -> fp32 [rows, D], labels_ptr -> int32 [rows] (raw
    device addresses, e.g. torch.Tensor.data_ptr()).  Asynchronous on `stream`.  Speaker bounds as in
    predict(); speakers_ptr (device int32 [U], 0 = none) receives the cluster counts.

    n_best=k (predict_device_sweep under the model's own pair): labels_ptr -> int32 [k][rows]; scores_ptr -> float32
    [U][k] (required), nbest_speakers_ptr -> int32 [U][k] and count_ptr -> int32 [U] (0 = none); speakers_ptr is
    ignored."""
    if n_best is not None:
      self.predict_device_sweep(x_ptr, frame_offsets, labels_ptr, scores_ptr, None, beam_size, look_ahead,
                                test_iteration, kcap, n_ctas, stream, lanes, cluster, engine, max_speakers,
                                min_speakers, n_best, nbest_speakers_ptr, count_ptr)
      return
    off = np.ascontiguousarray(frame_offsets, dtype=np.int64)
    mx, mn = speaker_bounds(len(off) - 1, max_speakers, min_speakers)
    ip = C.POINTER(C.c_int32)
    opts = self._opts(beam_size, look_ahead, test_iteration, kcap, n_ctas, lanes, cluster, engine)
    rc = self._lib.uis_predict_device_bounded(self._h, C.c_void_p(x_ptr),
                                              off.ctypes.data_as(C.POINTER(C.c_int64)), len(off) - 1,
                                              C.byref(opts), C.c_void_p(labels_ptr), None,
                                              C.c_void_p(stream),
                                              mx.ctypes.data_as(ip) if mx is not None else None,
                                              mn.ctypes.data_as(ip) if mn is not None else None,
                                              C.c_void_p(speakers_ptr))
    _check(self._lib, rc)

  def predict_sweep(self, seqs, decode_params, beam_size=10, look_ahead=1, test_iteration=2, kcap=0, n_ctas=0,
                    trace_utt=None, stream=0, lanes=0, cluster=0, engine=0, max_speakers=None, min_speakers=None,
                    n_best=1):
    """predict() under C (crp_alpha, transition_bias) pairs in one call (uis_predict_sweep).  Returns (labels, scores,
    speakers, count): labels[u] int32 [C][k][N_u], scores float32 [C][U][k], speakers int32 [C][U][k], count int32
    [C][U]; config c's entries are what predict(..., n_best=k) returns for a model created with pair c.  trace_utt
    names a job (c * U + u); the taps' final_scores / final_k are [C * U][...].  decode_params=None is the model's
    own pair (C = 1); n_best=None runs as 1."""
    n = len(seqs)
    dp, keep_dp, nc = self._sweep(decode_params)
    mx, mn = speaker_bounds(n, max_speakers, min_speakers)
    k = 1 if n_best is None else check_n_best(n_best, beam_size)
    keep, lens, offs = self._rows(seqs)
    # one flat int32 output buffer; the per-utterance pointers are base + 4 * offsets (no per-utterance allocation)
    flat = np.empty(max(nc * k * int(offs[-1]), 1), np.int32)
    outs = [flat[nc * k * offs[i]:nc * k * offs[i + 1]] for i in range(n)]
    out_addr = (flat.ctypes.data + 4 * nc * k * offs[:max(n, 1)]).astype(np.uint64)
    in_addr = np.fromiter((s.ctypes.data for s in keep), dtype=np.uint64, count=n) if n else np.zeros(1, np.uint64)
    opts = self._opts(beam_size, look_ahead, test_iteration, kcap, n_ctas, lanes, cluster, engine)
    taps, bufs, tp = None, None, None
    if trace_utt is not None:
      taps, bufs = self._taps(trace_utt, n * nc, [int(lens[j % max(n, 1)]) for j in range(n * nc)], beam_size,
                              look_ahead, test_iteration, kcap)
      tp = C.byref(taps)
    ip = C.POINTER(C.c_int32)
    scores = np.empty((nc, max(n, 1), k), np.float32)
    spk = np.empty((nc, max(n, 1), k), np.int32)
    count = np.empty((nc, max(n, 1)), np.int32)
    nb = NBestOut(out_addr.ctypes.data_as(C.POINTER(C.c_void_p)), None, scores.ctypes.data_as(C.POINTER(C.c_float)),
                  spk.ctypes.data_as(ip), count.ctypes.data_as(ip))
    arg = lambda a: a.ctypes.data_as(ip) if a is not None else None
    _check(self._lib, self._lib.uis_predict_sweep(
        self._h, in_addr.ctypes.data_as(C.POINTER(C.c_void_p)), lens.ctypes.data_as(C.POINTER(C.c_int64)), n,
        C.byref(opts), tp, C.c_void_p(stream), arg(mx), arg(mn), k, C.byref(nb), C.byref(dp)))
    del keep_dp
    # (a list of U utterances is held as [C][U][k]; with n == 0 the padding row is dropped)
    out = ([o.reshape(nc, k, int(lens[i])) for i, o in enumerate(outs)], scores[:, :n], spk[:, :n], count[:, :n])
    return (out, _trim_taps(bufs, trace_utt)) if bufs is not None else out

  def predict_device_sweep(self, x_ptr, frame_offsets, labels_ptr, scores_ptr, decode_params, beam_size=10,
                           look_ahead=1, test_iteration=2, kcap=0, n_ctas=0, stream=0, lanes=0, cluster=0, engine=0,
                           max_speakers=None, min_speakers=None, n_best=1, speakers_ptr=0, count_ptr=0):
    """Device-resident sweep (uis_predict_device_sweep): labels_ptr -> int32 [C][k][rows], scores_ptr -> float32
    [C][U][k] (required), speakers_ptr -> int32 [C][U][k], count_ptr -> int32 [C][U] (0 = none).  Asynchronous on
    `stream`.  decode_params=None is the model's own pair (C = 1)."""
    off = np.ascontiguousarray(frame_offsets, dtype=np.int64)
    dp, keep_dp, _ = self._sweep(decode_params)
    mx, mn = speaker_bounds(len(off) - 1, max_speakers, min_speakers)
    k = check_n_best(n_best, beam_size)
    ip = C.POINTER(C.c_int32)
    opts = self._opts(beam_size, look_ahead, test_iteration, kcap, n_ctas, lanes, cluster, engine)
    nb = NBestOut(None, C.c_void_p(labels_ptr), C.cast(C.c_void_p(scores_ptr), C.POINTER(C.c_float)),
                  C.cast(C.c_void_p(speakers_ptr), ip), C.cast(C.c_void_p(count_ptr), ip))
    _check(self._lib, self._lib.uis_predict_device_sweep(
        self._h, C.c_void_p(x_ptr), off.ctypes.data_as(C.POINTER(C.c_int64)), len(off) - 1, C.byref(opts), None,
        C.c_void_p(stream), mx.ctypes.data_as(ip) if mx is not None else None,
        mn.ctypes.data_as(ip) if mn is not None else None, k, C.byref(nb), C.byref(dp)))
    del keep_dp

  def score(self, seqs, labels, per_frame=False):
    """neg_likelihood of given labellings: seqs is a list of float64 [N_u, D] arrays (host), labels a list of
    canonical int label sequences (0, 1, 2, ... in order of first appearance), one of length N_u per utterance.
    Returns float32 scores [U]; with per_frame, (scores, list of float32 [N_u] per-frame increments).  This is
    score_sweep() under the model's own pair."""
    out = self.score_sweep(seqs, labels, None, per_frame)
    return (out[0][0], [f[0] for f in out[1]]) if per_frame else out[0]

  def score_sweep(self, seqs, labels, decode_params, per_frame=False):
    """score() under C (crp_alpha, transition_bias) pairs in one call (uis_score_sweep): float32 scores [C][U]; with
    per_frame, (scores, list of float32 [C][N_u] per-frame increments).  decode_params=None is the model's own pair
    (C = 1)."""
    if not isinstance(seqs, (list, tuple)) or not isinstance(labels, (list, tuple)):
      raise TypeError('seqs and labels must be lists')
    if len(seqs) != len(labels):
      raise ValueError('{} utterances but {} label sequences'.format(len(seqs), len(labels)))
    dp, keep_dp, nc = self._sweep(decode_params)
    n = len(seqs)
    keep, lens, _ = self._rows(seqs)
    labs = [np.ascontiguousarray(l, dtype=np.int32) for l in labels]
    for u, (s, l) in enumerate(zip(keep, labs)):
      if l.ndim != 1 or len(l) != s.shape[0]:
        raise ValueError('utterance {}: {} labels for {} frames'.format(u, l.size, s.shape[0]))
    scores = np.zeros((nc, max(n, 1)), np.float32)
    frames = [np.empty((nc, s.shape[0]), np.float32) for s in keep] if per_frame else None
    ptrs = lambda arrs: (C.c_void_p * max(len(arrs), 1))(*[a.ctypes.data for a in arrs])
    _check(self._lib, self._lib.uis_score_sweep(
        self._h, C.cast(ptrs(keep), C.POINTER(C.c_void_p)), lens.ctypes.data_as(C.POINTER(C.c_int64)), n,
        C.cast(ptrs(labs), C.POINTER(C.c_void_p)), scores.ctypes.data_as(C.POINTER(C.c_float)),
        C.cast(ptrs(frames), C.POINTER(C.c_void_p)) if per_frame else None, None, C.byref(dp)))
    del keep_dp
    return (scores[:, :n], frames) if per_frame else scores[:, :n]

  def score_device_sweep(self, x_ptr, frame_offsets, labels_ptr, scores_ptr, decode_params, frame_ptr=0, stream=0):
    """Device-resident score sweep (uis_score_device_sweep): scores_ptr -> float32 [C][U], frame_ptr -> float32
    [C][rows] (0 = none).  decode_params=None is the model's own pair (C = 1)."""
    off = np.ascontiguousarray(frame_offsets, dtype=np.int64)
    dp, keep_dp, _ = self._sweep(decode_params)
    _check(self._lib, self._lib.uis_score_device_sweep(
        self._h, C.c_void_p(x_ptr), off.ctypes.data_as(C.POINTER(C.c_int64)), len(off) - 1, C.c_void_p(labels_ptr),
        C.c_void_p(scores_ptr), C.c_void_p(frame_ptr), C.c_void_p(stream), C.byref(dp)))
    del keep_dp

  def score_device_ids(self, x_ptr, frame_offsets, ids_ptr, scores_ptr, decode_params, frame_ptr=0, labels_ptr=0,
                       stream=0):
    """Device-resident score sweep of arbitrary ids (uis_score_device_ids): ids_ptr -> int64 [rows], any values per
    frame, renamed in order of first appearance per utterance on the device; scores_ptr -> float32 [C][U], frame_ptr ->
    float32 [C][rows] (0 = none), labels_ptr -> int32 [rows] receives the canonical labels (0 = none).  Enqueues on
    `stream` without reading anything back.  decode_params=None is the model's own pair (C = 1)."""
    off = np.ascontiguousarray(frame_offsets, dtype=np.int64)
    dp, keep_dp, _ = self._sweep(decode_params)
    _check(self._lib, self._lib.uis_score_device_ids(
        self._h, C.c_void_p(x_ptr), off.ctypes.data_as(C.POINTER(C.c_int64)), len(off) - 1, C.c_void_p(ids_ptr),
        C.c_void_p(scores_ptr), C.c_void_p(frame_ptr), C.c_void_p(labels_ptr), C.c_void_p(stream), C.byref(dp)))
    del keep_dp

  def score_device(self, x_ptr, frame_offsets, labels_ptr, scores_ptr, frame_ptr=0, stream=0):
    """Device-resident variant: x_ptr -> fp32 [rows, D], labels_ptr -> canonical int32 [rows], scores_ptr -> float32
    [U], frame_ptr -> float32 [rows] per-frame increments (0 = none); raw device addresses.  Reads the labels back once
    to plan the chains, then enqueues the kernels on `stream` without waiting.  This is score_device_sweep() under the
    model's own pair, whose [1][U] / [1][rows] outputs are these layouts."""
    self.score_device_sweep(x_ptr, frame_offsets, labels_ptr, scores_ptr, None, frame_ptr, stream)

  def stats(self):
    s = Stats()
    _check(self._lib, self._lib.uis_get_stats(self._h, C.byref(s)))
    return s.as_dict()


def _gather_plan(index_lists):
  """(flat int32 row indices of every sub-sequence back to back, int64 offsets [n_sub + 1]) for set_corpus*."""
  offsets = np.zeros(len(index_lists) + 1, np.int64)
  np.cumsum([len(ix) for ix in index_lists], out=offsets[1:])
  flat = (np.concatenate(index_lists) if len(index_lists) else np.zeros(0)).astype(np.int32)
  return flat, offsets


class NativeTrainer:
  """Owns a `uis_trainer*`: parameters, gradients and Adam state of one fit_concatenated call live
  on the device; `step()` runs one iteration on a host batch.  `params`: dict name -> ndarray in
  param_order(depth) (rnn_init_hidden flattened to [depth * H]); hparams may carry rnn_depth (default 1),
  rnn_dropout (default 0) and dropout_seed."""

  def __init__(self, params, hparams, device=0):
    lib = load_library()
    self._lib = lib
    self._h = C.c_void_p()
    self.depth = int(hparams.get('rnn_depth', 1) or 1)
    self.order = param_order(self.depth)
    self.shapes = [tuple(np.asarray(params[k]).shape) for k in self.order]
    arrs = [_f32(np.asarray(params[k]).reshape(-1)) for k in self.order]
    self.H = int(np.asarray(params['linear_mean1.weight']).shape[0])
    self.D = int(np.asarray(params['linear_mean2.weight']).shape[0])
    ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    hp = TrainHParams(float(hparams['learning_rate']), float(hparams['sigma_alpha']),
                      float(hparams['sigma_beta']), float(hparams['regularization_weight']),
                      float(hparams['grad_max_norm']), int(bool(hparams['train_sigma2'])), self.depth,
                      float(hparams.get('rnn_dropout', 0.0) or 0.0), int(hparams.get('dropout_seed', 0) or 0))
    self._corpus = None
    _check(lib, lib.uis_trainer_create(C.byref(self._h), device, self.D, self.H, ptrs, C.byref(hp)))

  def close(self):
    if getattr(self, '_h', None) is not None and self._h:
      self._lib.uis_trainer_destroy(self._h)
      self._h = C.c_void_p()
    self._corpus = None  # the rows a set_corpus_device left the trainer reading

  def __del__(self):
    try:
      self.close()
    except Exception:  # pylint: disable=broad-except
      pass

  def losses(self, count):
    """(count, 3) array: losses of the last `count` steps, oldest first (synchronises)."""
    out = np.zeros((count, 3), np.float32)
    if count:
      _check(self._lib, self._lib.uis_trainer_losses(self._h, count, out.ctypes.data_as(C.POINTER(C.c_float))))
    return out

  def set_corpus(self, rows, index_lists):
    """rows: float64 [N, D] concatenated training sequence; index_lists: one int array of row indices per
    sub-sequence (utils.resize_indices).  Everything is copied to the device once."""
    rows = np.ascontiguousarray(rows, dtype=np.float64)
    assert rows.ndim == 2 and rows.shape[1] == self.D
    flat, offsets = _gather_plan(index_lists)
    _check(self._lib, self._lib.uis_trainer_set_corpus(
        self._h, rows.ctypes.data_as(C.c_void_p), rows.shape[0], flat.ctypes.data_as(C.c_void_p), len(flat),
        offsets.ctypes.data_as(C.c_void_p), len(index_lists)))
    self._corpus = None

  def set_corpus_device(self, tensors, index_lists, stream=0):
    """tensors: torch CUDA tensors [N_i, D] on the trainer's device, all float32, float16, bfloat16 or float64, any strides;
    row indices refer to their rows back to back.  The trainer reads the rows in place at every step_corpus, so they
    must not change until close() or the next set_corpus*.  The row-address table (8 bytes per row) is built by torch
    on the current stream; a tensor whose elements are not in unit stride is made contiguous first.  This object keeps
    the tensors, those copies and the table alive until then."""
    import torch
    code = {torch.float32: UIS_DTYPE_F32, torch.float16: UIS_DTYPE_F16, torch.bfloat16: UIS_DTYPE_BF16,
            torch.float64: UIS_DTYPE_F64}[tensors[0].dtype]
    with torch.no_grad():
      rows = [t.detach() if t.shape[1] == 1 or t.stride(1) == 1 else t.detach().contiguous() for t in tensors]
      device = rows[0].device
      n = sum(r.shape[0] for r in rows)
      # (from pinned memory, so the copy is ordered on the current stream without the host waiting for that stream)
      meta = torch.tensor([[r.data_ptr(), r.stride(0) * r.element_size(), r.shape[0]] for r in rows],
                          dtype=torch.int64).pin_memory().to(device, non_blocking=True)
      # address of row j of utterance u = base_u + (j - first row of u) * row stride_u
      utt = torch.repeat_interleave(torch.arange(len(rows), device=device), meta[:, 2], output_size=n)
      first = torch.cumsum(meta[:, 2], 0) - meta[:, 2]
      table = meta[utt, 0] + (torch.arange(n, device=device) - first[utt]) * meta[utt, 1]
    flat, offsets = _gather_plan(index_lists)
    _check(self._lib, self._lib.uis_trainer_set_corpus_device(
        self._h, C.c_void_p(table.data_ptr()), code, n, flat.ctypes.data_as(C.c_void_p), len(flat),
        offsets.ctypes.data_as(C.c_void_p), len(index_lists), C.c_void_p(stream)))
    self._corpus = (rows, table, meta)

  def step_corpus(self, chosen, mode=0, want_losses=False, stream=0):
    """One iteration on sub-sequences `chosen` (ids in column order, lengths descending).  mode as in
    uis_trainer_step; asynchronous unless want_losses."""
    ids = np.ascontiguousarray(chosen, dtype=np.int32)
    losses = np.zeros(3, np.float32) if want_losses else None
    _check(self._lib, self._lib.uis_trainer_step_corpus(
        self._h, ids.ctypes.data_as(C.c_void_p), len(ids), mode,
        losses.ctypes.data_as(C.POINTER(C.c_float)) if want_losses else None, C.c_void_p(stream)))
    return tuple(float(v) for v in losses) if want_losses else None

  def comm_size(self):
    return int(self._lib.uis_trainer_comm_size(self._h))

  def step_shard(self, rnn_input, lengths, stream=0):
    """Data-parallel shard: forward + backward with un-normalised gradients (mode 2)."""
    x = _f32(rnn_input)
    L, B, D = x.shape
    lens = np.ascontiguousarray(lengths, dtype=np.int32)
    _check(self._lib, self._lib.uis_trainer_step(self._h, x.ctypes.data_as(C.c_void_p),
                                                  lens.ctypes.data_as(C.POINTER(C.c_int32)), B, L, 2, None,
                                                  C.c_void_p(stream)))

  def comm_export(self, dev_ptr, stream=0):
    _check(self._lib, self._lib.uis_trainer_comm_export(self._h, C.c_void_p(dev_ptr), C.c_void_p(stream)))

  def comm_apply(self, dev_ptr, stream=0):
    _check(self._lib, self._lib.uis_trainer_comm_apply(self._h, C.c_void_p(dev_ptr), C.c_void_p(stream)))

  def step_async(self, rnn_input, lengths, stream=0):
    """Enqueues one full iteration and returns immediately (losses via `losses()`)."""
    x = _f32(rnn_input)
    L, B, D = x.shape
    assert D == self.D
    lens = np.ascontiguousarray(lengths, dtype=np.int32)
    _check(self._lib, self._lib.uis_trainer_step(self._h, x.ctypes.data_as(C.c_void_p),
                                                  lens.ctypes.data_as(C.POINTER(C.c_int32)), B, L, 0, None,
                                                  C.c_void_p(stream)))

  def step(self, rnn_input, lengths, grads_only=False, stream=0):
    """rnn_input: float32 [L, B, D] zero-padded time-major batch; lengths: [B] descending.
    Returns (loss1, loss2, loss3)."""
    x = _f32(rnn_input)
    L, B, D = x.shape
    assert D == self.D
    lens = np.ascontiguousarray(lengths, dtype=np.int32)
    losses = np.zeros(3, np.float32)
    rc = self._lib.uis_trainer_step(self._h, x.ctypes.data_as(C.c_void_p),
                                    lens.ctypes.data_as(C.POINTER(C.c_int32)), B, L,
                                    1 if grads_only else 0, losses.ctypes.data_as(C.POINTER(C.c_float)),
                                    C.c_void_p(stream))
    _check(self._lib, rc)
    return tuple(float(v) for v in losses)

  def _get(self, what):
    outs = [np.empty(int(np.prod(s)) if s else 1, np.float32) for s in self.shapes]
    ptrs = (C.c_void_p * len(outs))(*[o.ctypes.data for o in outs])
    _check(self._lib, self._lib.uis_trainer_get(self._h, what, ptrs))
    return {k: o.reshape(s) for k, o, s in zip(self.order, outs, self.shapes)}

  def parameters(self):
    return self._get(0)

  def gradients(self):
    return self._get(1)
