"""Compiler check of the fp16 flood kernel's tile epilogue (no GPU needed, only nvcc).

After a tile's MMAs the two consumer warpgroups run the epilogue: neighbour exchange, masks, bias, residual, fp16
stores.  The tensor cores sit idle while it runs, and eight warps share the SM's four issue slots, so its length is
time.  The row geometry (inside the FoV, x == 0, x == fx - 1) comes from a per-engine table loaded under the MMAs
rather than from a float decode of the row index, and addresses are formed once per tile.

The region checked runs from the wait that ends a tile's run of 18 HGMMA to the branch back to the next tile's
mbarrier wait.  It holds one body per epilogue kind (EPI_A, EPI_B_FIRST, EPI_B, EPI_LAST), which end in branches to
a common join.  Before the row-flag table and the per-tile addresses, every body had 315-378 instructions, 4 of them
F2I.TRUNC; now the three conv-layer kinds have 173-230 (the first body also holds the dispatch) and EPI_LAST, which
also runs conv_lom and the step counts, 289-291.  The bounds leave some headroom above those counts."""

import os
import re
import shutil
import subprocess

import pytest

from ffn_b200 import build

pytestmark = pytest.mark.slow

kMaxBodyInstructions = 250       # EPI_A, EPI_B_FIRST, EPI_B
kMaxLastBodyInstructions = 320   # EPI_LAST: the body with the four-lane conv_lom sum (SHFL.BFLY)

_INS = re.compile(r'/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;')
_BRA = re.compile(r'^(@!?U?P\w+\s+)?BRA(?:\.\w+)*\s+(0x[0-9a-f]+)$')


def _tool(name):
  nvcc = build.nvcc_path()
  cand = os.path.join(os.path.dirname(nvcc), name) if os.path.isabs(nvcc) else shutil.which(name)
  return cand if cand and os.path.exists(cand) else None


def instructions(sass_lines):
  """[(address, text)] of one function's SASS listing."""
  out = []
  for line in sass_lines:
    m = _INS.search(line)
    if m:
      out.append((int(m.group(1), 16), m.group(2)))
  return out


def branch(text):
  """(predicated, target address) of a BRA, else None."""
  m = _BRA.match(text)
  if not m:
    return None
  return bool(m.group(1)), int(m.group(2), 16)


def epilogue_bodies(ins):
  """For every wait that ends a run of >= 18 HGMMA: the epilogue bodies that follow it, as lists of instruction texts.

  The region ends at the first branch back to an address before the wait (the tile loop's back edge).  Inside it,
  unconditional forward branches to a common target close the bodies; that target (the join) closes the last one."""
  regions = []
  run = 0
  for i, (addr, text) in enumerate(ins):
    if 'HGMMA.64x96x16' in text:
      run += 1
      continue
    if 'WARPGROUP.DEPBAR' not in text:
      continue
    if run >= 18:
      end = next(j for j in range(i + 1, len(ins)) if (b := branch(ins[j][1])) and b[1] <= addr)
      back_target = branch(ins[end][1])[1]
      waits = [t for a, t in ins if back_target <= a < addr and 'SYNCS.PHASECHK' in t]
      assert waits, 'the back edge at %#x does not lead to a tile wait' % ins[end][0]
      region = ins[i:end + 1]
      exits = [(k, branch(t)[1]) for k, (_, t) in enumerate(region) if (b := branch(t)) and not b[0] and b[1] > addr]
      join = max({tgt for _, tgt in exits}, key=lambda tgt: sum(1 for _, x in exits if x == tgt))
      cuts = [k for k, tgt in exits if tgt == join] + [next(k for k, (a, _) in enumerate(region) if a == join)]
      bodies, start = [], 0
      for k in cuts:
        bodies.append([t for _, t in region[start:k + 1]])
        start = k + 1
      regions.append((region, bodies))
    run = 0
  return regions


@pytest.fixture(scope='module')
def plain_fp16_epilogues(tmp_path_factory):
  nvcc, cuobjdump = _tool('nvcc'), _tool('cuobjdump')
  if nvcc is None or cuobjdump is None:
    pytest.skip('nvcc / cuobjdump not found')
  cubin = str(tmp_path_factory.mktemp('epilogue') / 'engine.cubin')
  res = subprocess.run([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '--default-stream',
                        'per-thread', '-cubin', '-o', cubin, build.SRC], capture_output=True, text=True)
  assert res.returncode == 0, res.stderr[-4000:]
  sass = subprocess.run([cuobjdump, '-sass', cubin], capture_output=True, text=True, check=True).stdout
  # ffn_flood_kernel<false> of the product namespace (<true> is the split-fp16 parity instance)
  funcs = [f for f in re.split(r'\n\s*Function : ', sass) if f.startswith('_ZN3ffn5plain16ffn_flood_kernelILb0E')]
  assert len(funcs) == 1
  regions = epilogue_bodies(instructions(funcs[0].splitlines()))
  assert regions, 'no run of 18 HGMMA followed by an epilogue'
  return regions


def test_epilogue_has_no_float_int_conversion(plain_fp16_epilogues):
  for region, _ in plain_fp16_epilogues:
    conv = ['%#x %s' % (a, t) for a, t in region if re.search(r'\b(F2I|I2F|I2FP)\b', t)]
    assert not conv, conv


def test_epilogue_bodies_are_short(plain_fp16_epilogues):
  for _, bodies in plain_fp16_epilogues:
    sizes = [len(b) for b in bodies]
    assert len(bodies) == 4, sizes   # EPI_A, EPI_B_FIRST, EPI_B, EPI_LAST
    last = [i for i, b in enumerate(bodies) if any('SHFL.BFLY' in t for t in b)]
    assert len(last) == 1, sizes
    assert sizes[last[0]] <= kMaxLastBodyInstructions, sizes
    assert max(n for i, n in enumerate(sizes) if i != last[0]) <= kMaxBodyInstructions, sizes
