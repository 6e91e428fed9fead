"""Builds libffn_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'csrc', 'engine.cu')
OUT = os.path.join(HERE, 'libffn_b200.so')
DEPS = [os.path.join(HERE, 'csrc', f) for f in os.listdir(os.path.join(HERE, 'csrc'))] + [
    os.path.join(os.path.dirname(HERE), 'include', 'ffn_b200.h')]


def nvcc_path():
  for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
    if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
      return cand
  return 'nvcc'


def up_to_date():
  if not os.path.exists(OUT):
    return False
  t = os.path.getmtime(OUT)
  return all(os.path.getmtime(d) <= t for d in DEPS)


def build(force=False, verbose=False):
  """Builds the engine library."""
  if not force and up_to_date():
    return OUT
  tmp = OUT + '.tmp%d' % os.getpid()   # linked next to the target and renamed over it: a reader never sees a partial file
  cmd = [
      nvcc_path(), '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17', '--default-stream', 'per-thread',
      '-Xcompiler', '-fPIC', '-shared', '-o', tmp, SRC, '-lcudart',
  ]
  if verbose:
    cmd.insert(1, '-Xptxas')
    cmd.insert(2, '-v')
  res = subprocess.run(cmd, capture_output=True, text=True)
  if res.returncode != 0:
    if os.path.exists(tmp):
      os.unlink(tmp)
    raise RuntimeError('nvcc failed:\n%s\n%s' % (res.stdout, res.stderr))
  os.replace(tmp, OUT)
  if verbose:
    sys.stderr.write(res.stderr)
  return OUT


if __name__ == '__main__':
  print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
