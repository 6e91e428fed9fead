"""Split-consensus fixture: the REAL reference `ffn/inference/consensus.py`, `segmentation.py` and `storage.py`,
unmodified.

    PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION=python python tests/golden/make_golden_consensus.py

Harness as in make_golden_storage.py: third-party imports stubbed, TensorFlow's gfile replaced by os / open.  What
the modules are given besides, and nothing else:
  * `connectomics.segmentation.labels` -> a module whose every attribute raises when it is called: the paths pinned
    here (split consensus, loading with `split_cc: false`) never reach connected components;
  * `ffn.inference.consensus_pb2` -> this package's runtime-built `ConsensusRequest` (the reference's generated file
    predates the current protobuf runtime).

Cases of `compute_consensus_for_segmentations` (inputs, `split_min_size`, the returned array with its dtype and `v1`
after the call, or the name of the exception): min_size 0, 1 and one that drops fragments; equal-count ties between
two b ids; (a, 0) pairs kept and (0, b) pairs dropped; ids >= 2^32 and >= 2^63 in `a` with and without 0, ids >= 2^32
in `b`; `a` all zero; `a == b`; results reduced to uint8, uint16, uint32 and uint64; a shape mismatch, a wrong dtype
in either input, and an unsupported consensus type.
Cases of `compute_consensus`: two seg-*.npz written by the reference's `save_subvolume` at corner (4, 8, 12), loaded
through `load_segmentation_from_source` with `split_cc: false` plain, with `threshold` (a .prob file) and with a
coordinate-expression mask; the first file's origins include keys above its max id, one of which a new split id takes.
Output: consensus_ref.npz.
"""
import contextlib
import os
import shutil
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

OUT = os.path.join(HERE, 'consensus_ref.npz')
CORNER = (4, 8, 12)
U64 = np.uint64


class _Unreachable(types.ModuleType):
  def __getattr__(self, name):
    if name.startswith('__'):
      raise AttributeError(name)

    def fail(*a, **k):
      raise AssertionError('connectomics.segmentation.labels.%s was called' % name)
    return fail


def reference_modules():
  os.environ.setdefault('PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION', 'python')
  mg.install_stubs()
  labels = _Unreachable('connectomics.segmentation.labels')
  sys.modules['connectomics.segmentation.labels'] = labels
  sys.modules['connectomics.segmentation'].labels = labels
  sys.path.insert(0, mg.REF)
  from ffn.inference import storage as ref_storage
  from ffn.inference import segmentation as ref_segmentation
  assert ref_segmentation.labels is labels
  from ffn_b200.inference import consensus_pb2
  sys.modules['ffn.inference.consensus_pb2'] = consensus_pb2
  sys.modules['ffn.inference'].consensus_pb2 = consensus_pb2
  from ffn.inference import consensus as ref_consensus
  assert ref_consensus.consensus_pb2 is consensus_pb2 and ref_consensus.storage is ref_storage

  class _GFileCtx:
    def __init__(self, path, mode='r'):
      self._f = open(path, mode)

    def __enter__(self):
      return self._f

    def __exit__(self, *a):
      self._f.close()

  class _Gfile:
    makedirs = staticmethod(lambda p: os.makedirs(p, exist_ok=True))
    exists = staticmethod(os.path.exists)
    GFile = _GFileCtx
  ref_storage.gfile = _Gfile

  @contextlib.contextmanager
  def atomic_file(path, mode='w+b'):
    with open(path, mode) as f:
      yield f
  ref_storage.atomic_file = atomic_file
  return ref_consensus, ref_storage, consensus_pb2


def blocks(shape, cell, seed, offset=0, ids=None):
  """Box cells of edge `cell` with ids from `ids` (or 1..), jittered by a seeded random shift."""
  rng = np.random.RandomState(seed)
  z, y, x = np.indices(shape)
  sz, sy, sx = rng.randint(0, cell, 3)
  k = ((z + sz) // cell) * 1000 + ((y + sy) // cell) * 100 + (x + sx) // cell + offset
  _, lab = np.unique(k, return_inverse=True)
  lab = lab.reshape(shape).astype(U64) + U64(1)
  if ids is not None:
    lab = np.asarray(ids, U64)[(lab - U64(1)).astype(np.int64) % len(ids)]
  return lab


def split_cases():
  """(tag, a, b, min_size, type) per case."""
  shape = (12, 14, 16)
  a = blocks(shape, 5, 1)
  b = blocks(shape, 4, 2)
  rng = np.random.RandomState(3)
  a_zero = a.copy()
  a_zero[rng.rand(*shape) < 0.1] = 0
  b_zero = b.copy()
  b_zero[rng.rand(*shape) < 0.1] = 0
  cases = [('min0', a_zero, b_zero, 0), ('min1', a_zero, b_zero, 1), ('min_drop', a_zero, b_zero, 9)]

  # ties: a = 5 overlaps b = 7 and b = 3 with 6 voxels each and b = 9 with 4; a = 8 overlaps b = 2 and b = 1 with 7
  a_t = np.zeros((1, 4, 8), U64)
  b_t = np.zeros((1, 4, 8), U64)
  a_t[0, :2, :8] = 5
  b_t[0, :2, :3] = 7
  b_t[0, :2, 3:6] = 3
  b_t[0, :2, 6:8] = 9
  a_t[0, 2:, :] = 8
  b_t[0, 2:, :4] = 2
  b_t[0, 2:, 4:] = 1
  a_t[0, 3, 7] = 0
  a_t[0, 2, 0] = 0
  cases.append(('ties', a_t, b_t, 0))

  # (a, 0) kept, (0, b) dropped
  a_z = a.copy()
  b_z = b.copy()
  b_z[:, :, :5] = 0
  a_z[:, :4, :] = 0
  cases.append(('zero_pairs', a_z, b_z, 2))

  big = 2**32 + 7
  huge = 2**63 + 11
  ids_big = [big + 5 * k for k in range(60)]
  cases.append(('a_ge_2_32_with_0', np.where(a_zero > 0, np.asarray(ids_big, U64)[(a_zero % U64(60)).astype(np.int64)],
                                             U64(0)), b_zero, 0))
  cases.append(('a_ge_2_63_no_0', blocks(shape, 5, 1, ids=[huge + 3 * k for k in range(40)] + [17, 2**40]), b, 1))
  cases.append(('b_ge_2_32', a_zero, blocks(shape, 4, 2, ids=[0, 2**35 + 1, 2**35, 2**50, 3, 2**64 - 1]), 0))
  cases.append(('a_all_zero', np.zeros(shape, U64), b, 0))
  cases.append(('a_equals_b', b_zero.copy(), b_zero.copy(), 0))

  # reduce_id_bits: every id below 256, above 255, above 65535, above 2^32 - 1 after the split
  cases.append(('reduce_u8', (a % U64(7)) + U64(1), (b % U64(5)), 0))
  cases.append(('reduce_u16', a + U64(250), b, 0))
  cases.append(('reduce_u32', a + U64(65530), b, 0))
  cases.append(('reduce_u64', a + U64(2**32 - 5), b, 0))
  return [c + (2,) for c in cases] + [
      ('err_shape', a, b[:, :, :-1], 0, 2),
      ('err_dtype_a', a.astype(np.int64), b, 0, 2),
      ('err_dtype_b', a, b.astype(np.uint32), 0, 2),
      ('err_type', a, b, 0, 3),
  ]


def write_sources(ref_storage, root):
  """Two seg-*.npz by the reference's save_subvolume, a .prob for the first, and the sources of each loading mode."""
  shape = (10, 12, 14)
  rng = np.random.RandomState(5)
  v1 = blocks(shape, 5, 7, ids=[3, 17, 40, 9])
  v1[rng.rand(*shape) < 0.05] = 0
  v2 = blocks(shape, 4, 8)
  origins1 = {k: ref_storage.OriginInfo((k % 10, 2, 3), 10 + k, 0.5 * k) for k in (3, 9, 17, 40, 41, 44)}
  origins2 = {int(k): ref_storage.OriginInfo((1, 1, 1), 1, 0.1) for k in np.unique(v2)}
  d1, d2 = os.path.join(root, 'forward'), os.path.join(root, 'reverse')
  ref_storage.save_subvolume(v1, origins1, ref_storage.segmentation_path(d1, CORNER))
  ref_storage.save_subvolume(v2, origins2, ref_storage.segmentation_path(d2, CORNER))
  qprob = rng.randint(1, 256, shape).astype(np.uint8)
  prob_path = ref_storage.object_prob_path(d1, CORNER)
  with open(prob_path, 'wb') as f:
    np.savez_compressed(f, qprob=qprob)
  return d1, d2


def main():
  ref_consensus, ref_storage, consensus_pb2 = reference_modules()
  out = {}
  cases = split_cases()
  out['n_split'] = len(cases)
  for i, (tag, a, b, min_size, ctype) in enumerate(cases):
    a_in, b_in = a.copy(), b.copy()
    request = consensus_pb2.ConsensusRequest(split_min_size=min_size)
    if ctype != 2:
      request = types.SimpleNamespace(type=ctype, split_min_size=min_size)   # a closed proto2 enum rejects 3
    v1 = a.copy()
    error, res = '', np.zeros(0, U64)
    try:
      res = ref_consensus.compute_consensus_for_segmentations(v1, b, request)
    except (ValueError, TypeError) as e:
      error = type(e).__name__
    assert np.array_equal(b, b_in)
    print('%-18s %-10s %s' % (tag, error or res.dtype, '' if error else '%d ids' % np.unique(res).size))
    out.update({'tag_%d' % i: tag, 'a_%d' % i: a_in, 'b_%d' % i: b_in, 'min_size_%d' % i: min_size,
                'type_%d' % i: ctype, 'error_%d' % i: error, 'out_%d' % i: res, 'v1_after_%d' % i: v1})

  tmp = tempfile.mkdtemp(prefix='consensus_golden_')
  d1, d2 = write_sources(ref_storage, tmp)
  files = {}
  for name, path in (('seg1', ref_storage.segmentation_path(d1, CORNER)), ('prob1', ref_storage.object_prob_path(d1, CORNER)),
                     ('seg2', ref_storage.segmentation_path(d2, CORNER))):
    with open(path, 'rb') as f:
      files[name] = np.frombuffer(f.read(), np.uint8)
    out['file_%s' % name] = files[name]
    out['relpath_%s' % name] = os.path.relpath(path, tmp)
  from ffn_b200.inference import protos
  modes = [('plain', {}), ('threshold', {'threshold': 0.6}),
           ('mask', {'mask': 'x + 2 * y > 52'}), ('mask_threshold', {'threshold': 0.3, 'mask': 'z < 7'})]
  out['n_consensus'] = len(modes)
  out['corner'] = np.array(CORNER)
  for i, (tag, kw) in enumerate(modes):
    request = protos.ConsensusRequest(split_min_size=2 if i % 2 else 0)
    request.segmentation1.directory = d1
    request.segmentation1.split_cc = False
    request.segmentation2.directory = d2
    request.segmentation2.split_cc = False
    request.segmentation2.min_size = 0
    if 'threshold' in kw:
      request.segmentation1.threshold = kw['threshold']
    if 'mask' in kw:
      request.segmentation1.mask.masks.add().coordinate_expression.expression = kw['mask']
    l1, o1 = ref_storage.load_segmentation_from_source(request.segmentation1, CORNER)
    l2, o2 = ref_storage.load_segmentation_from_source(request.segmentation2, CORNER)
    seg, origins = ref_consensus.compute_consensus(CORNER, request)
    keys = sorted(origins)
    stale = [k for k in keys if int(k) > int(l1.max())]
    print('consensus %-15s %s %d ids, origins %s (above the loaded max id: %s)' % (
        tag, seg.dtype, np.unique(seg).size, [int(k) for k in keys], [int(k) for k in stale]))
    out.update({
        'ctag_%d' % i: tag, 'split_min_size_%d' % i: request.split_min_size,
        'threshold_%d' % i: kw.get('threshold', np.nan), 'mask_%d' % i: kw.get('mask', ''),
        'loaded1_%d' % i: l1, 'loaded2_%d' % i: l2,
        'loaded1_origin_ids_%d' % i: np.array(sorted(int(k) for k in o1), U64),
        'seg_%d' % i: seg, 'origin_ids_%d' % i: np.array([int(k) for k in keys], U64),
        'origin_start_%d' % i: np.array([origins[k].start_zyx for k in keys], np.int64).reshape(-1, 3),
        'origin_iters_%d' % i: np.array([origins[k].iters for k in keys], np.int64),
        'origin_wall_%d' % i: np.array([origins[k].walltime_sec for k in keys], np.float64),
        'stale_%d' % i: np.array([int(k) for k in stale], U64)})
  shutil.rmtree(tmp)
  np.savez_compressed(OUT, **out)
  print('wrote', OUT)


if __name__ == '__main__':
  main()
