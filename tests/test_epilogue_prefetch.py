"""Compiler check of the fp16 flood kernel's residual prefetch (no GPU needed, only nvcc).

The epilogue of an odd layer reads the tile's fp32 residual rows.  The kernel prefetches them into L1 just before it
issues the tile's MMAs, so that the L2 round trip runs under the tensor-core work instead of after it.  In SASS the
prefetch is `CCTL.E.PF1`; it must come after the previous tile's wait (`WARPGROUP.DEPBAR`) and before the tile's run
of HGMMAs."""

import os
import re
import shutil
import subprocess

import pytest

from ffn_b200 import build

pytestmark = pytest.mark.slow


def _tool(name):
  nvcc = build.nvcc_path()
  cand = os.path.join(os.path.dirname(nvcc), name) if os.path.isabs(nvcc) else shutil.which(name)
  return cand if cand and os.path.exists(cand) else None


@pytest.fixture(scope='module')
def plain_fp16_sass(tmp_path_factory):
  nvcc, cuobjdump = _tool('nvcc'), _tool('cuobjdump')
  if nvcc is None or cuobjdump is None:
    pytest.skip('nvcc / cuobjdump not found')
  cubin = str(tmp_path_factory.mktemp('prefetch') / 'engine.cubin')
  res = subprocess.run([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '--default-stream',
                        'per-thread', '-cubin', '-o', cubin, build.SRC], capture_output=True, text=True)
  assert res.returncode == 0, res.stderr[-4000:]
  sass = subprocess.run([cuobjdump, '-sass', cubin], capture_output=True, text=True, check=True).stdout
  # ffn_flood_kernel<false> of the product namespace (<true> is the split-fp16 parity instance)
  funcs = [f for f in re.split(r'\n\s*Function : ', sass) if f.startswith('_ZN3ffn5plain16ffn_flood_kernelILb0E')]
  assert len(funcs) == 1
  return funcs[0].splitlines()


def test_residual_prefetch_is_issued_before_each_tile_of_mmas(plain_fp16_sass):
  runs = []          # for every run of >= 18 HGMMA between two waits: prefetches seen before its first HGMMA
  prefetches = before = run = 0
  for line in plain_fp16_sass:
    if 'HGMMA.64x96x16' in line:
      if run == 0:
        before = prefetches
      run += 1
    elif 'CCTL.E.PF1' in line and run == 0:
      prefetches += 1
    elif 'WARPGROUP.DEPBAR' in line:
      if run >= 18:
        runs.append(before)
      prefetches = run = 0
  assert runs, 'no run of 18 HGMMA'
  assert all(n >= 2 for n in runs), runs   # rows m0 and m0 + 8 of the thread
