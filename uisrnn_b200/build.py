"""Builds libuisrnn_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

Staleness is decided by a content hash of the sources (a sidecar file next to the library), not
by mtimes -- the tree is copied to the GPU box, which does not preserve a meaningful mtime order --
and the build runs under a file lock so that several ranks started together do not race.
"""
import fcntl
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libuisrnn_b200.so')
STAMP = LIB + '.srchash'
SOURCES = ['uis_api.cu', 'uis_train.cu', 'uis_kernels_beam_large.cu', 'uis_kernels_beam_small.cu', 'uis_kernels_beam_cluster.cu', 'uis_kernels_beam_stat.cu', 'uis_kernels_beam_tc.cu',
           'uis_kernels_tree_large.cu', 'uis_kernels_tree_small.cu', 'uis_kernels_score.cu', 'uis_score_plan.cu']
DEPS = SOURCES + ['uis_beam.cuh', 'uis_beam_tc.cuh', 'uis_beam_stat.cuh', 'uis_beam_tree.cuh', 'uis_prepass.cuh', 'uis_common.cuh', 'uis_launch.cuh',
        os.path.join('..', '..', 'include', 'uisrnn_b200.h')]
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
              '-shared', '-Xcompiler', '-fPIC', '--threads', '0']


def find_nvcc():
  for cand in (os.environ.get('NVCC'), shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
    if cand and os.path.exists(cand):
      return cand
  raise RuntimeError('nvcc not found')


def source_hash():
  h = hashlib.sha256()
  h.update(' '.join(NVCC_FLAGS).encode())
  for dep in DEPS:
    with open(os.path.join(CSRC, dep), 'rb') as f:
      h.update(dep.encode())
      h.update(f.read())
  return h.hexdigest()


def is_stale():
  if not os.path.exists(LIB) or not os.path.exists(STAMP):
    return True
  with open(STAMP) as f:
    return f.read().strip() != source_hash()


def build(force=False, verbose=False):
  if not force and not is_stale():
    return LIB
  with open(LIB + '.lock', 'w') as lock:
    fcntl.flock(lock, fcntl.LOCK_EX)
    try:
      if not force and not is_stale():   # another process built it while we waited
        return LIB
      tmp = LIB + '.tmp.%d' % os.getpid()
      cmd = [find_nvcc()] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + \
          ['-o', tmp] + [os.path.join(CSRC, s) for s in SOURCES]
      res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
      if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError('nvcc failed: ' + ' '.join(cmd))
      if verbose:
        sys.stderr.write(res.stderr)
      os.replace(tmp, LIB)
      with open(STAMP, 'w') as f:
        f.write(source_hash())
    finally:
      fcntl.flock(lock, fcntl.LOCK_UN)
  return LIB


if __name__ == '__main__':
  print(build(force='--force' in sys.argv, verbose=True))
