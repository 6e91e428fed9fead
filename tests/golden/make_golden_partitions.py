"""Partition-map fixture: the REAL reference `compute_partitions.py`, loaded by path and unmodified, with the
reference's own `ffn/inference/segmentation.py`, `storage.py` and `ffn/utils/bounding_box.py`.

    PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION=python python tests/golden/make_golden_partitions.py

Third-party imports are stubbed by make_golden.install_stubs(); absl is the real package.  What the script is given
besides, and nothing else:
  * `_TupleIndexing`, an ndarray subclass whose `__getitem__` turns a list of slices into a tuple, as numpy before
    1.23 did: `compute_partitions` indexes `seg_array[valid_sel]` and `object_mask[valid_sel]` with a list, which
    current numpy rejects.  The input array is passed as a view of this class, so `clear_dust` still writes into it;
  * `_H5File`, a minimal in-memory `h5py.File` (datasets with `attrs`, `create_dataset` with `fillvalue`) standing
    in for h5py in both the script's `main` and the reference storage's volume masks;
  * as in make_golden_build_mask.py, storage's un-vendored `connectomics.common.bounding_box` -> the reference's own
    `ffn/utils/bounding_box.BoundingBox` with its module-level `intersection` as a method (volume-mask clipping).

Cases of `compute_partitions` (inputs, the returned corner and array, `seg_array` after the call, or the name of the
exception): iso, anisotropic and zero radii on an axis; unsorted and single thresholds; `min_size` 0, 1 and one that
removes objects; a whitelist with absent ids and 0; exclusion spheres partly outside the VALID region with integer
and float values; a coordinate-expression mask and a volume mask; ids >= 2^32, >= 2^63 and negative int64; all-zero
input, one label everywhere, and a volume smaller than the LOM; empty thresholds with and without labels.
Case of `main`: an input with `bounding_boxes` attrs, one of which vanishes once adjusted, run with the flags the
script can parse (no mask, whitelist or exclusions); the written dataset and its attrs.
Output: partitions_ref.npz.
"""
import importlib.util
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

OUT = os.path.join(HERE, 'partitions_ref.npz')
# A volume mask's source in the stored MaskConfigs text; the tests substitute a file of their own.
MASK_PLACEHOLDER = '@MASK@'
THRESHOLDS = [0.025, 0.05, 0.075, 0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9]


class _TupleIndexing(np.ndarray):
  def __getitem__(self, key):
    if isinstance(key, list) and all(isinstance(k, slice) for k in key):
      key = tuple(key)
    return super().__getitem__(key)


class _Dataset:
  def __init__(self, data):
    self.data = data
    self.attrs = {}

  shape = property(lambda self: self.data.shape)
  ndim = property(lambda self: self.data.ndim)
  dtype = property(lambda self: self.data.dtype)

  def __getitem__(self, key):
    return self.data[key]

  def __setitem__(self, key, value):
    self.data[key] = value


_FILES = {}


class _H5File:
  def __init__(self, path, mode='r'):
    if mode == 'w':
      _FILES[path] = {}
    self._d = _FILES[path]

  def __enter__(self):
    return self

  def __exit__(self, *a):
    return False

  def __getitem__(self, name):
    return self._d[name]

  def create_dataset(self, name, shape, dtype, fillvalue=0, **unused):
    ds = _Dataset(np.full(shape, fillvalue, dtype))
    self._d[name] = ds
    return ds


def reference_script():
  os.environ.setdefault('PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION', 'python')
  mg.install_stubs()
  h5 = types.ModuleType('h5py')
  h5.File = _H5File
  sys.modules['h5py'] = h5
  sys.path.insert(0, mg.REF)
  from ffn.inference import storage as ref_storage
  ref_storage.h5py = h5
  from ffn.utils import bounding_box as ref_bbox

  class _BBox(ref_bbox.BoundingBox):
    def intersection(self, other):
      return ref_bbox.intersection(self, other)
  ref_storage.bounding_box = types.SimpleNamespace(BoundingBox=_BBox)
  spec = importlib.util.spec_from_file_location('ref_compute_partitions', os.path.join(mg.REF, 'compute_partitions.py'))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  assert mod.h5py is h5 and mod.storage is ref_storage
  from ffn.inference import inference_pb2
  return mod, inference_pb2


def voronoi(shape, n, seed, dtype=np.int64, ids=None, zero_frac=0.0):
  """Nearest-site labels 1..n (or ids[k]) on `shape`, with a seeded fraction of voxels set to 0."""
  rng = np.random.RandomState(seed)
  sites = rng.rand(n, 3) * np.asarray(shape)
  grid = np.stack(np.indices(shape), -1).reshape(-1, 1, 3).astype(np.float64)
  lab = np.argmin(((grid - sites[None]) ** 2).sum(-1), axis=1).reshape(shape)
  out = (np.asarray(ids, dtype)[lab] if ids is not None else (lab + 1).astype(dtype))
  if zero_frac:
    out[rng.rand(*shape) < zero_frac] = 0
  return out


def cases():
  """(tag, seg, thresholds, lom_radius, id_whitelist, exclusion_regions, mask_text, mask_volume, min_size)."""
  base = voronoi((14, 18, 22), 9, 1, zero_frac=0.05)
  th = THRESHOLDS
  c = [
      ('iso', base, th, [3, 3, 3], None, None, '', None, 0),
      ('aniso', base, th, [4, 2, 1], None, None, '', None, 0),
      ('zero_x', base, th, [0, 2, 3], None, None, '', None, 0),
      ('zero_all', base, th, [0, 0, 0], None, None, '', None, 0),
      ('zero_zy', base, th, [2, 0, 0], None, None, '', None, 1),
      ('unsorted', base, [0.5, 0.1, 0.9, 0.3], [2, 3, 2], None, None, '', None, 0),
      ('single', base, [0.4], [2, 2, 2], None, None, '', None, 0),
      ('min1', base, th, [2, 2, 2], None, None, '', None, 1),
  ]
  dusty = base.copy()
  dusty[3:5, 4:6, 5:8] = 40
  dusty[10, 10, 10] = 41
  dusty[0, 0, :3] = 42
  c.append(('min_drop', dusty, th, [2, 2, 2], None, None, '', None, 13))
  c.append(('whitelist', base, th, [2, 1, 2], [3, 0, 5, 77, 8, 2**40], None, '', None, 0))
  c.append(('excl_int', base, th, [2, 2, 2], None, [(3, 4, 5, 4), (20, 1, 0, 6), (-2, 30, 20, 9)], '', None, 0))
  c.append(('excl_float', base, th, [2, 2, 1], None, [(3.5, 4, 5.25, 4.5), (10, 8, 6, 2.0), (21.7, 17.2, 13.1, 3.3)],
            '', None, 0))
  c.append(('mask_expr', base, th, [2, 2, 2], None, None,
            'masks { coordinate_expression { expression: "(x + 2 * y > 40) & (z < 6)" } }', None, 0))
  mvol = np.zeros((1,) + base.shape, np.uint8)   # (channel, z, y, x), as the reference's volume masks read it
  mvol[0, 7, 3:9, 2:4] = 3
  mvol[0, 12, 15, 20] = 9
  c.append(('mask_volume', base, th, [1, 2, 3], None, [(4, 4, 4, 2)],
            'masks { volume { mask { hdf5: "%s" } channels { channel: 0 min_value: 2 max_value: 5 } } }'
            % MASK_PLACEHOLDER, mvol, 0))
  big = voronoi((12, 13, 15), 7, 2, np.uint64, ids=[2**32 + 3, 2**33, 5, 2**63 + 9, 2**64 - 1, 2**63, 2**32 + 4])
  c.append(('u64_big', big, th, [2, 2, 2], None, None, '', None, 1))
  c.append(('u64_big_white', big, th, [2, 2, 2], [2**63 + 9, 5, 2**64 - 1, 7], None, '', None, 0))
  neg = voronoi((12, 13, 15), 6, 3, np.int64, ids=[-1, -2**63, 4, -7, 2**62, 9])
  neg[:2, :2, :2] = -5
  c.append(('i64_neg', neg, th, [2, 1, 2], None, None, '', None, 4))
  c.append(('i64_neg_white', neg, th, [2, 1, 2], [-7, 4, -2**63, -3], None, '', None, 0))
  c.append(('u8_labels', base.astype(np.uint8), th, [1, 1, 1], None, None, '', None, 30))
  c.append(('all_zero', np.zeros((8, 9, 10), np.int32), th, [1, 1, 1], None, [(2, 2, 2, 1)], '', None, 5))
  c.append(('one_label', np.full((8, 9, 10), 7, np.uint16), th, [2, 1, 3], None, None, '', None, 10))
  c.append(('smaller_than_lom', base[:3, :4, :5].copy(), th, [3, 3, 3], None, None, '', None, 0))
  c.append(('smaller_one_axis', base[:, :, :5].copy(), th, [3, 2, 1], None, None, '', None, 0))
  c.append(('empty_thresholds', base, [], [1, 1, 1], None, None, '', None, 0))
  c.append(('empty_thresholds_no_labels', np.zeros((5, 6, 7), np.int64), [], [1, 1, 1], None, None, '', None, 0))
  c.append(('empty_thresholds_whitelist', base, [], [1, 1, 1], [999], None, '', None, 0))
  return c


def pack_regions(regions):
  """Exclusion regions as (values float64 [n, 4], is_int bool [n, 4]); an empty array with has_* False for None."""
  if regions is None:
    return np.zeros((0, 4)), np.zeros((0, 4), bool)
  vals = np.array([[float(v) for v in r] for r in regions], np.float64).reshape(-1, 4)
  is_int = np.array([[isinstance(v, int) for v in r] for r in regions], bool).reshape(-1, 4)
  return vals, is_int


def main():
  mod, inference_pb2 = reference_script()
  from google.protobuf import text_format
  out = {}
  cs = cases()
  out['n_cases'] = len(cs)
  out['mask_placeholder'] = MASK_PLACEHOLDER
  for i, (tag, seg, th, radius, white, regions, mask_text, mask_volume, min_size) in enumerate(cs):
    mask_configs = None
    if mask_text:
      mask_configs = inference_pb2.MaskConfigs()
      text_format.Parse(mask_text.replace(MASK_PLACEHOLDER, 'mask.h5:m'), mask_configs)
      if mask_volume is not None:
        _H5File('mask.h5', 'w').create_dataset('m', mask_volume.shape, mask_volume.dtype)[...] = mask_volume
    arr = seg.copy()
    error, corner, res = '', np.zeros(3, np.int64), np.zeros((0, 0, 0), np.uint8)
    try:
      corner, res = mod.compute_partitions(arr.view(_TupleIndexing), list(th), list(radius), white, regions,
                                           mask_configs, min_size)
    except (IndexError, ValueError, TypeError, OverflowError, AssertionError) as e:
      error = type(e).__name__
    assert type(res) is np.ndarray and res.dtype == np.uint8
    vals, is_int = pack_regions(regions)
    print('%-28s %-12s %s' % (tag, error or str(res.shape), '' if error else np.unique(res)))
    out.update({'tag_%d' % i: tag, 'seg_%d' % i: seg, 'thresholds_%d' % i: np.array(th, np.float64),
                'lom_radius_%d' % i: np.array(radius, np.int64), 'has_whitelist_%d' % i: white is not None,
                'whitelist_%d' % i: np.array([int(w) for w in white or []], object).astype(str),
                'has_regions_%d' % i: regions is not None, 'regions_%d' % i: vals, 'regions_int_%d' % i: is_int,
                'mask_text_%d' % i: mask_text, 'has_mask_volume_%d' % i: mask_volume is not None,
                'mask_volume_%d' % i: mask_volume if mask_volume is not None else np.zeros(0, np.uint8),
                'min_size_%d' % i: min_size, 'error_%d' % i: error, 'corner_%d' % i: np.asarray(corner),
                'out_%d' % i: res, 'seg_after_%d' % i: arr})

  # main: flags the script parses as given (thresholds, radius, min_size), on an input with bounding_boxes attrs.
  seg = voronoi((16, 18, 20), 8, 4, np.uint32, zero_frac=0.02)
  bboxes = np.array([[(0, 0, 0), (20, 18, 16)], [(3, 4, 5), (4, 3, 6)], [(10, 2, 1), (9, 14, 12)]], np.int64)
  ds = _H5File('in.h5', 'w').create_dataset('stack', seg.shape, seg.dtype)
  ds.data = seg.copy().view(_TupleIndexing)
  ds.attrs['bounding_boxes'] = bboxes
  argv = ['compute_partitions.py', '--input_volume=in.h5:stack', '--output_volume=out.h5:af',
          '--thresholds=0.1,0.3,0.5,0.7,0.9', '--lom_radius=3,2,2', '--min_size=40']
  mod.FLAGS(argv)
  mod.main([])
  res = _FILES['out.h5']['af']
  print('main', res.shape, res.attrs['partition_counts'].tolist())
  out.update({'main_seg': seg, 'main_bboxes': bboxes, 'main_argv': np.array(argv[1:]), 'main_out': res.data,
              'main_out_bboxes': np.array(res.attrs['bounding_boxes'], np.int64),
              'main_partition_counts': np.asarray(res.attrs['partition_counts'])})
  np.savez_compressed(OUT, **out)
  print('wrote', OUT)


if __name__ == '__main__':
  main()
