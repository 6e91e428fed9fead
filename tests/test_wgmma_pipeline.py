"""Compiler checks of the flood kernel's tensor-core pipeline (no GPU needed, only nvcc).

ptxas decides for a whole function whether its wgmma instructions may stay in flight together; when it
cannot prove that, it waits for every MMA before issuing the next one (and says so on -v).  The fp16
kernel issues 18 MMAs per consumer warpgroup and tile, which must reach the tensor core back to back."""

import re

import pytest

import flood_cubins

pytestmark = pytest.mark.slow


def _is_fp16_flood_kernel(mangled):
  # ffn_flood_kernel<true> is the split-fp16 parity instance
  return 'ffn_flood_kernel' in mangled and 'ILb1E' not in mangled


@pytest.fixture(scope='module')
def compiled():
  return flood_cubins.flood_kernels()


def test_fp16_flood_kernels_not_serialized(compiled):
  log, _ = compiled
  names = re.findall(r"function '(\w+)'", '\n'.join(l for l in log.splitlines() if 'instructions are serialized' in l))
  assert not [n for n in names if _is_fp16_flood_kernel(n)], log


def test_fp16_flood_kernels_do_not_spill(compiled):
  log, _ = compiled
  props = re.findall(r'Function properties for (\w+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads',
                     log)
  fp16 = [p for p in props if _is_fp16_flood_kernel(p[0])]
  assert len(fp16) == 2, props
  for name, _, stores, loads in fp16:
    assert (stores, loads) == ('0', '0'), name


def test_plain_fp16_kernel_issues_a_tile_of_mmas_without_waiting(compiled):
  _, sass = compiled
  funcs = re.split(r'\n\s*Function : ', sass)
  plain = [f for f in funcs if f.startswith('_ZN3ffn5plain') and _is_fp16_flood_kernel(f.split('\n', 1)[0])]
  assert len(plain) == 1
  longest = run = 0
  for line in plain[0].splitlines():
    if 'HGMMA.64x96x16' in line:
      run += 1
      longest = max(longest, run)
    elif 'WARPGROUP.DEPBAR' in line:
      run = 0
  assert longest >= 18, longest
