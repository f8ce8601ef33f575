"""Installs the unmodified reference (google/uis-rnn) into the git-ignored oracle/_ref/.

bench.py's `cpu_baseline` and `--impl reference` legs time the original project's own predict() from there; without
it they time the numpy port oracle/uis_oracle.py and say so (`kind: "port"`).  The reference is pure Python, so the
"build" is a copy of its `uisrnn` package, made once.  The source is a checkout of google/uis-rnn named by
$UISRNN_REFERENCE_DIR, by default /root/reference; where that directory does not exist nothing happens.
"""
import os
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
DST = os.path.join(HERE, '_ref')


def build(src=None):
  """Returns the install directory, or None when there is neither an install nor a source to make one from."""
  if os.path.exists(os.path.join(DST, 'uisrnn', 'uisrnn.py')):
    return DST
  src = src or os.environ.get('UISRNN_REFERENCE_DIR') or '/root/reference'
  pkg = os.path.join(src, 'uisrnn')
  if not os.path.exists(os.path.join(pkg, 'uisrnn.py')):
    return None
  try:
    os.makedirs(DST, exist_ok=True)
    tmp = tempfile.mkdtemp(dir=DST)  # copy next to the target, then rename: a reader never sees half a package
    try:
      # plain file copies: a read-only checkout must not make the copy read-only (renaming a directory needs write
      # permission on it)
      shutil.copytree(pkg, os.path.join(tmp, 'uisrnn'), copy_function=shutil.copyfile,
                      ignore=shutil.ignore_patterns('__pycache__', '*.pyc'))
      for d, _, _ in os.walk(os.path.join(tmp, 'uisrnn')):
        os.chmod(d, 0o755)
      try:
        os.rename(os.path.join(tmp, 'uisrnn'), os.path.join(DST, 'uisrnn'))
      except OSError:  # another process installed it first
        if not os.path.exists(os.path.join(DST, 'uisrnn', 'uisrnn.py')):
          raise
    finally:
      shutil.rmtree(tmp, ignore_errors=True)
  except OSError as err:
    sys.stderr.write('oracle/_ref: could not install the reference from %s (%s); bench.py will time the numpy port\n'
                     % (src, err))
    return None
  return DST


if __name__ == '__main__':
  print(build(sys.argv[1] if len(sys.argv) > 1 else None))
