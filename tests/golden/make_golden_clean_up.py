"""Connected-component clean-up fixture: the REAL reference `ffn/inference/segmentation.py` `clean_up` and
`clean_up_and_count`, unmodified.

    PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION=python python tests/golden/make_golden_clean_up.py

Harness as in make_golden_consensus.py: third-party imports stubbed.  The module's one third-party call,
`connectomics.segmentation.labels.split_disconnected_components`, is not vendored, so it is given here by its
definition, what skimage.measure.label(labels, connectivity=c, background=0) returns: a component is a maximal set of
voxels of one non-zero id connected under scipy.ndimage.generate_binary_structure(ndim, c), components are numbered
1, 2, ... in C order of their first voxel, 0 stays 0, and a connectivity outside [1, ndim] raises ValueError.  It is
written as a plain breadth-first search and shares no code with oracle/clean_up.py.

Cases (input, arguments, the array after the call, each returned dict as sorted keys and values with their types, or
the name of the exception): connectivity 1 / 2 / 3 on diagonal-only contacts, checkerboards and 26-only corner
touches; one id in several pieces and one id everywhere; min_size 0, 1, a component's size and one above; a dusted
voxel before the first zero of the input; ids >= 2^32 and >= 2^63; all-zero and empty input; an axis of length 1,
2-D and 1-D input; split_cc=False with and without min_size; every compute_id_map / compute_counts / return_id_map
combination; connectivity 0, 4 and above ndim.
Output: clean_up_ref.npz.
"""
import collections
import itertools
import os
import sys
import types

import numpy as np
from scipy import ndimage

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

OUT = os.path.join(HERE, 'clean_up_ref.npz')
U64 = np.uint64


def split_disconnected_components(labels, connectivity=1):
  if not 1 <= connectivity <= labels.ndim:
    raise ValueError('Connectivity for %dD image should be in [1, ..., %d]. Got %r.' % (
        labels.ndim, labels.ndim, connectivity))
  structure = ndimage.generate_binary_structure(labels.ndim, connectivity)
  centre = np.ones(labels.ndim, int)
  offsets = [tuple(np.array(o) - centre) for o in zip(*np.nonzero(structure)) if tuple(o) != tuple(centre)]
  out = np.zeros(labels.shape, np.int64)
  n = 0
  for start in itertools.product(*[range(s) for s in labels.shape]):
    if labels[start] == 0 or out[start]:
      continue
    n += 1
    out[start] = n
    queue = collections.deque([start])
    while queue:
      p = queue.popleft()
      for o in offsets:
        q = tuple(a + b for a, b in zip(p, o))
        if all(0 <= q[k] < labels.shape[k] for k in range(labels.ndim)) and not out[q] and labels[q] == labels[start]:
          out[q] = n
          queue.append(q)
  return out


def reference_segmentation():
  os.environ.setdefault('PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION', 'python')
  mg.install_stubs()
  labels = types.ModuleType('connectomics.segmentation.labels')
  labels.split_disconnected_components = split_disconnected_components
  sys.modules['connectomics.segmentation.labels'] = labels
  sys.modules['connectomics.segmentation'].labels = labels
  sys.path.insert(0, mg.REF)
  from ffn.inference import segmentation as ref_segmentation
  assert ref_segmentation.labels is labels
  return ref_segmentation


def cases():
  """(tag, seg, function, kwargs) per case."""
  out = []

  def add(tag, seg, fn='clean_up_and_count', **kw):
    out.append((tag, np.asarray(seg, U64), fn, kw))

  # diagonal-only contacts: 5 touches along an xy edge (18), then a corner (26); 9 is a separate 6-connected bar
  d = np.zeros((3, 4, 5), U64)
  d[0, 0, 0] = d[0, 1, 1] = d[1, 2, 2] = d[1, 2, 3] = 5
  d[2, :, 4] = 9
  d[2, 0, 3] = 9
  for c in (1, 2, 3):
    add('diagonal_c%d' % c, d, connectivity=c)
  cb = ((np.indices((4, 4, 4)).sum(0) % 2) + 1).astype(U64)
  for c in (1, 2, 3):
    add('checker3d_c%d' % c, cb, connectivity=c)
  cb2 = ((np.indices((5, 6)).sum(0) % 2) * 3).astype(U64)
  for c in (1, 2):
    add('checker2d_c%d' % c, cb2, connectivity=c)
  # two cubes of one id touching only at a corner, and two of another touching along an edge
  k = np.zeros((4, 4, 8), U64)
  k[:2, :2, :2] = 4
  k[2:, 2:, 2:4] = 4
  k[:2, :2, 4:6] = 6
  k[:2, 2:, 6:8] = 6
  for c in (1, 2, 3):
    add('corner26_c%d' % c, k, connectivity=c)

  rng = np.random.RandomState(11)
  r = rng.randint(0, 4, (6, 7, 8)).astype(U64) * U64(3)
  r[rng.rand(6, 7, 8) < 0.3] = 7   # 7 everywhere, in many pieces
  for c in (1, 2, 3):
    add('pieces_c%d' % c, r, connectivity=c)
  add('one_id', np.full((4, 5, 6), 42, U64))
  add('one_id_min_drop', np.full((4, 5, 6), 42, U64), min_size=121)

  # min_size: 0, 1, equal to a component's size (kept), one above (dusted)
  m = np.zeros((4, 6, 6), U64)
  m[:2, :2, :2] = 8          # 8 voxels
  m[2:, 3:, 3:] = 8          # 18 voxels, a second piece of 8
  m[:, 4:, :2] = 2           # 16
  m[0, 5, 5] = 3             # 1
  for ms in (0, 1, 8, 9, 16, 17):
    add('min_size_%d' % ms, m, min_size=ms)
  add('min_size_float', m, min_size=8.5)
  add('min_size_negative', m, min_size=-3)

  # a dusted voxel before the first zero of the input: the 0 row of the id map names the dusted id
  f = np.full((3, 4, 5), 4, U64)
  f[0, 0, 0] = 8
  f[2, 1, 1:3] = 0
  add('dust_before_zero', f, min_size=2)
  add('dust_before_zero_no_split', f, split_cc=False, min_size=2)

  big, huge = 2**32 + 5, 2**63 + 9
  add('ids_ge_2_32', np.where(r > 0, r * U64(2**31) + U64(big), U64(0)), connectivity=2, min_size=2)
  add('ids_ge_2_63', np.where(r > 0, r + U64(huge), U64(0)), connectivity=3)
  add('ids_max', np.where(r == 7, U64(2**64 - 1), r), min_size=3)

  add('all_zero', np.zeros((3, 4, 5), U64))
  add('all_zero_bad_connectivity', np.zeros((3, 4, 5), U64), connectivity=0)
  add('empty', np.zeros((0, 4, 5), U64))
  add('axis_len_1', r[:1], connectivity=3)
  add('two_d_c1', r[2], connectivity=1)
  add('two_d_c2', r[2], connectivity=2, min_size=2)
  add('one_d', r[2, 3], connectivity=1)
  add('no_split', r, split_cc=False)
  add('no_split_min_size', r, split_cc=False, min_size=3)

  for cm, cc in itertools.product((False, True), repeat=2):
    add('compute_%d%d' % (cm, cc), r, connectivity=2, min_size=2, compute_id_map=cm, compute_counts=cc)
  for rim in (False, True):
    add('clean_up_map_%d' % rim, r, 'clean_up', min_size=2, return_id_map=rim)
  add('clean_up_no_split', r, 'clean_up', split_cc=False, min_size=2, return_id_map=True)

  add('err_connectivity_0', r, connectivity=0)
  add('err_connectivity_4', r, connectivity=4)
  add('err_connectivity_2d', r[2], connectivity=3)
  add('err_connectivity_1d', r[2, 3], connectivity=2)
  return out


def dict_arrays(d):
  """(kind, sorted keys, values, key type name, value type name) of a returned dict or None."""
  if d is None:
    return 'None', np.zeros(0, U64), np.zeros(0, U64), '', ''
  keys = sorted(d)
  ktypes = {type(k).__name__ for k in keys}
  vtypes = {type(d[k]).__name__ for k in keys}
  assert len(ktypes) <= 1 and len(vtypes) <= 1, (ktypes, vtypes)
  vals = [d[k] for k in keys]
  return ('dict', np.array(keys, U64), np.array(vals, np.asarray(vals).dtype if vals else U64),
          ktypes.pop() if ktypes else '', vtypes.pop() if vtypes else '')


def main():
  ref = reference_segmentation()
  out = {}
  cs = cases()
  out['n'] = len(cs)
  for i, (tag, seg, fn, kw) in enumerate(cs):
    work = seg.copy()
    error, res = '', None
    try:
      res = getattr(ref, fn)(work, **kw)
    except (ValueError, TypeError) as e:
      error = type(e).__name__
    if fn == 'clean_up':
      maps = (res, None)
    else:
      maps = res if res is not None else (None, None)
    rec = {'tag': tag, 'fn': fn, 'kwargs': repr(sorted(kw.items())), 'seg': seg, 'after': work, 'error': error}
    for name, d in zip(('map', 'counts'), maps):
      kind, keys, vals, kt, vt = dict_arrays(d)
      rec.update({name + '_kind': kind, name + '_keys': keys, name + '_vals': vals, name + '_ktype': kt,
                  name + '_vtype': vt})
    print('%-28s %-7s %s' % (tag, error or 'ok', '' if error else '%d ids' % np.unique(work).size))
    out.update({'%s_%d' % (k, i): v for k, v in rec.items()})
  np.savez_compressed(OUT, **out)
  print('wrote', OUT)


if __name__ == '__main__':
  main()
