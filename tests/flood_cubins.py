"""The flood kernel as the library compiles it, for the compiler checks (test_wgmma_pipeline.py, test_epilogue_sass.py,
test_epilogue_prefetch.py): flood_plain.cu and flood_profiled.cu compiled to cubins with the library's nvcc flags
plus -Xptxas -v, in parallel, once per test process."""

import functools
import os
import shutil
import subprocess
import tempfile
from concurrent.futures import ThreadPoolExecutor

import pytest

from ffn_b200 import build

SOURCES = ('flood_plain.cu', 'flood_profiled.cu')


def _tool(name):
  nvcc = build.nvcc_path()
  cand = os.path.join(os.path.dirname(nvcc), name) if os.path.isabs(nvcc) else shutil.which(name)
  return cand if cand and os.path.exists(cand) else None


@functools.lru_cache(maxsize=None)
def _compile():
  cuobjdump = _tool('cuobjdump')
  with tempfile.TemporaryDirectory() as tmp:

    def one(src):
      cubin = os.path.join(tmp, src + '.cubin')
      log = build.compile(os.path.join(build.CSRC, src), cubin, ['-cubin', '-Xptxas', '-v'])
      sass = subprocess.run([cuobjdump, '-sass', cubin], capture_output=True, text=True, check=True).stdout
      return log, sass

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as pool:
      logs, sass = zip(*pool.map(one, SOURCES))
  return '\n'.join(logs), '\n'.join(sass)


def flood_kernels():
  """(ptxas -v log, cuobjdump -sass listing) of the plain and the profiled flood kernels; skips without nvcc."""
  if _tool('nvcc') is None or _tool('cuobjdump') is None:
    pytest.skip('nvcc / cuobjdump not found')
  return _compile()
