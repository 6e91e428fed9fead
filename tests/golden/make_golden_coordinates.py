"""Training-coordinate fixture: the REAL reference `build_coordinates.py`, loaded by path and unmodified.

    PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION=python python tests/golden/make_golden_coordinates.py

Third-party imports are stubbed by make_golden.install_stubs(); absl is the real package, and `main` is driven
through the script's own FLAGS.  What the script is given besides, and nothing else:
  * a recording `tensorflow.compat.v1`: `train.Example/Features/Feature/Int64List/BytesList` build plain Python
    values, `SerializeToString` returns the Example itself, and `python_io.TFRecordWriter` (which must be given
    GZIP `TFRecordOptions`) collects the written Examples in order;
  * `_H5File`, the in-memory `h5py.File` of make_golden_partitions.py, holding the partition volumes.
`np.random.seed(seed)` is called right before `main`, which draws from numpy's global RandomState.

Cases: one volume with an anisotropic margin and values 0-13 and 255, at two seeds; two volumes of different shapes
and names, where some values are first seen in the second volume, also with two `main` calls after one seed (which
pins the number of draws); a partition of one voxel (repeated by np.resize) and one that lies only in the margin; an
all-255 volume next to a normal one; a margin that empties the smaller volume only; a margin of 0 (ValueError); a
non-ASCII name; and one larger volume.  Per case and call: each record's center (x, y, z) and the index of its
label_volume_name among the case's names.  Output: coordinates_ref.npz.
"""
import importlib.util
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402
from make_golden_partitions import _H5File  # noqa: E402

OUT = os.path.join(HERE, 'coordinates_ref.npz')
_WRITTEN = {}   # path -> [(center, name bytes)]


class _Example:
  def __init__(self, features):
    self.features = features

  def SerializeToString(self):
    return self


class _Writer:
  def __init__(self, path, options=None):
    assert options == ('TFRecordOptions', 'GZIP'), options
    self.path = path
    self.records = []

  def __enter__(self):
    return self

  def __exit__(self, *a):
    _WRITTEN[self.path] = self.records
    return False

  def write(self, ex):
    feat = ex.features
    assert sorted(feat) == ['center', 'label_volume_name']
    kind_c, center = feat['center']
    kind_n, name = feat['label_volume_name']
    assert kind_c == 'int64_list' and kind_n == 'bytes_list' and len(center) == 3 and len(name) == 1
    assert isinstance(name[0], bytes)
    self.records.append(([int(v) for v in center], name[0]))


def _feature(int64_list=None, bytes_list=None):
  assert (int64_list is None) != (bytes_list is None)
  return ('int64_list', int64_list) if int64_list is not None else ('bytes_list', bytes_list)


def recording_tf():
  tf = types.ModuleType('tensorflow.compat.v1')
  tf.train = types.SimpleNamespace(
      Example=lambda features: _Example(features), Features=lambda feature: dict(feature), Feature=_feature,
      Int64List=lambda value: list(value), BytesList=lambda value: list(value))
  tf.python_io = types.SimpleNamespace(
      TFRecordOptions=lambda compression: ('TFRecordOptions', compression),
      TFRecordCompressionType=types.SimpleNamespace(GZIP='GZIP'), TFRecordWriter=_Writer)
  return tf


def reference_script():
  os.environ.setdefault('PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION', 'python')
  mg.install_stubs()
  tf = recording_tf()
  sys.modules['tensorflow.compat.v1'] = tf
  sys.modules['tensorflow.compat'].v1 = tf
  h5 = types.ModuleType('h5py')
  h5.File = _H5File
  sys.modules['h5py'] = h5
  spec = importlib.util.spec_from_file_location('ref_build_coordinates', os.path.join(mg.REF, 'build_coordinates.py'))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  assert mod.h5py is h5 and mod.tf is tf
  return mod


def blocky(shape, values, seed, p255=0.0):
  """Partition-like uint8 volume: `values` in blocks of random sizes along each axis, a seeded fraction of 255."""
  rng = np.random.RandomState(seed)
  idx = [np.cumsum(rng.rand(s) < 0.35) for s in shape]
  v = np.asarray(values, np.uint8)
  out = v[(idx[0][:, None, None] * 7 + idx[1][None, :, None] * 3 + idx[2][None, None, :]) % v.size]
  if p255:
    out[rng.rand(*shape) < p255] = 255
  return out


def cases():
  """(tag, [(name, volume)], margin (z, y, x), seed, calls)."""
  aniso = blocky((20, 24, 28), range(14), 1, p255=0.08)
  a2 = blocky((18, 20, 22), [0, 1, 2, 3, 4, 5, 255], 2)
  b2 = blocky((14, 16, 12), range(3, 10), 3, p255=0.03)
  one = blocky((10, 12, 14), [1, 2], 4)
  one[5, 6, 7] = 7     # one voxel inside the crop
  one[0, 3, 3] = 9     # in the margin only: never seen
  normal = blocky((10, 11, 12), [0, 4, 8, 255], 5)
  large = blocky((30, 40, 48), range(12), 6, p255=0.02)
  return [
      ('aniso', [('vol', aniso)], (2, 3, 4), 0, 1),
      ('aniso_seed7', [('vol', aniso)], (2, 3, 4), 7, 1),
      ('two_volumes', [('alpha', a2), ('beta', b2)], (1, 2, 3), 3, 1),
      ('two_calls', [('alpha', a2), ('beta', b2)], (1, 2, 3), 11, 2),
      ('one_voxel', [('one', one)], (1, 1, 1), 5, 1),
      ('all_255', [('ignored', np.full((12, 12, 12), 255, np.uint8)), ('normal', normal)], (1, 1, 1), 6, 1),
      ('empty_smaller', [('big', aniso), ('small', one)], (5, 4, 3), 8, 1),
      ('margin_zero', [('vol', aniso)], (0, 2, 2), 9, 1),
      ('non_ascii', [('Zellkörper_体積', normal)], (2, 1, 3), 10, 1),
      ('large', [('large', large)], (3, 4, 5), 12, 1),
  ]


def main():
  mod = reference_script()
  out = {}
  cs = cases()
  out['n_cases'] = len(cs)
  total = 0
  for i, (tag, vols, margin, seed, calls) in enumerate(cs):
    specs = []
    for k, (name, vol) in enumerate(vols):
      path = 'part%d_%d.h5' % (i, k)
      _H5File(path, 'w').create_dataset('af', vol.shape, vol.dtype)[...] = vol
      specs.append('%s:%s:af' % (name, path))
    argv = ['build_coordinates.py', '--partition_volumes=' + ','.join(specs), '--coordinate_output=coords_%d' % i,
            '--margin=' + ','.join(str(m) for m in margin)]
    mod.FLAGS(argv)
    np.random.seed(seed)
    error = ''
    for c in range(calls):
      _WRITTEN.pop('coords_%d' % i, None)
      try:
        mod.main([])
      except ValueError as e:
        error = type(e).__name__
        assert 'coords_%d' % i not in _WRITTEN
        break
      recs = _WRITTEN['coords_%d' % i]
      names = [n.encode('utf-8') for n, _ in vols]
      out['centers_%d_%d' % (i, c)] = np.array([r[0] for r in recs], np.int32).reshape(-1, 3)
      out['name_index_%d_%d' % (i, c)] = np.array([names.index(r[1]) for r in recs], np.uint8)
      total += len(recs)
    print('%-14s %s' % (tag, error or [len(out['centers_%d_%d' % (i, c)]) for c in range(calls)]))
    out.update({'tag_%d' % i: tag, 'names_%d' % i: np.array([n for n, _ in vols]),
                'n_volumes_%d' % i: len(vols), 'margin_%d' % i: np.array(margin, np.int64), 'seed_%d' % i: seed,
                'calls_%d' % i: calls, 'error_%d' % i: error})
    for k, (_, vol) in enumerate(vols):
      out['volume_%d_%d' % (i, k)] = vol
  np.savez_compressed(OUT, **out)
  print('%d records; wrote %s' % (total, OUT))


if __name__ == '__main__':
  main()
