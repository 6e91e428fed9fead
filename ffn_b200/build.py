"""Builds libffn_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

Every csrc/*.cu is one translation unit; they compile in parallel and link into one shared library."""

import glob
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OUT = os.path.join(HERE, 'libffn_b200.so')
DEPS = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [
    os.path.join(os.path.dirname(HERE), 'include', 'ffn_b200.h')]
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17', '--default-stream', 'per-thread']


def nvcc_path():
  for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
    if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
      return cand
  return 'nvcc'


def compile(src, out, extra_flags=()):
  """Runs nvcc with FLAGS on src (a path, or a list of objects to link) into out; returns nvcc's messages."""
  srcs = [src] if isinstance(src, str) else list(src)
  res = subprocess.run([nvcc_path()] + FLAGS + ['-o', out] + srcs + list(extra_flags), capture_output=True, text=True)
  if res.returncode != 0:
    raise RuntimeError('nvcc failed on %s:\n%s\n%s' % (' '.join(map(os.path.basename, srcs)), res.stdout, res.stderr))
  return res.stdout + res.stderr


def up_to_date():
  if not os.path.exists(OUT):
    return False
  t = os.path.getmtime(OUT)
  return all(os.path.getmtime(d) <= t for d in DEPS)


def build(force=False, verbose=False):
  """Builds the engine library."""
  if not force and up_to_date():
    return OUT
  srcs = sorted(glob.glob(os.path.join(CSRC, '*.cu')))
  extra = ['-c', '-Xcompiler', '-fPIC'] + (['-Xptxas', '-v'] if verbose else [])
  tmp = OUT + '.tmp%d' % os.getpid()   # linked next to the target and renamed over it: a reader never sees a partial file
  with tempfile.TemporaryDirectory() as objdir:
    objs = [os.path.join(objdir, os.path.basename(s) + '.o') for s in srcs]
    with ThreadPoolExecutor(max_workers=len(srcs)) as pool:
      logs = list(pool.map(lambda so: compile(so[0], so[1], extra), zip(srcs, objs)))
    try:
      compile(objs, tmp, ['-shared', '-lcudart'])
    except Exception:
      if os.path.exists(tmp):
        os.unlink(tmp)
      raise
  os.replace(tmp, OUT)
  if verbose:
    sys.stderr.write(''.join(logs))
  return OUT


if __name__ == '__main__':
  print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
