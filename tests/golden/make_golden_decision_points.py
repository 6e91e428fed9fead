"""find_decision_points fixture: the REAL reference function (ffn/utils/decision_point.py:27-145, with
ffn/inference/segmentation.py's clean_up_and_count / clear_dust for optimize_sparse) on the volumes of its own unit
test (ffn/utils/tests/decision_point_test.py) and on Voronoi-cell phantoms.

    PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION=python python tests/golden/make_golden_decision_points.py

The reference modules run unmodified; pandas is used as installed.  The one un-vendored call,
connectomics.segmentation.labels.watershed_expand, is injected with its documented behaviour ("every empty voxel
gets the id of the nearest segment, up to max_distance"), defined as:
  edt = ndimage.distance_transform_edt(seg == 0, sampling=voxel_size[::-1]);
  expanded = the id of the nearest labelled voxel (same sampling), the smallest id when several are equally near;
  expanded = seg where edt > max_distance.
connectomics.common.bounding_box.BoundingBox is a box with start / size in (x, y, z) and to_slice3d().

Output: decision_points_ref.npz; per case the inputs (`_seg`, `_voxel_size`, `_max_distance` (nan: None), `_box`
(start xyz + size xyz, empty: None), `_optimize_sparse`, `_threshold`), the result in key order (`_ids` [n, 2]
uint64, `_dist`, `_points` [n, 3] int64 x, y, z) and the label array after the call (`_seg_after`).
"""
import os
import sys

import numpy as np
from scipy import ndimage

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402


class Box:
  def __init__(self, start, size):
    self.start, self.size = np.asarray(start, dtype=np.int64), np.asarray(size, dtype=np.int64)

  def to_slice3d(self):
    lo, hi = self.start, self.start + self.size
    return np.index_exp[lo[2]:hi[2], lo[1]:hi[1], lo[0]:hi[0]]


def watershed_expand_definition(seg, voxel_size, max_distance=None):
  sampling = tuple(float(v) for v in voxel_size)[::-1]
  edt = ndimage.distance_transform_edt(seg == 0, sampling=sampling)
  expanded = seg.copy()
  nearest = np.full(seg.shape, np.inf)
  for i in sorted(int(v) for v in np.unique(seg) if v != 0):
    d = ndimage.distance_transform_edt(seg != seg.dtype.type(i), sampling=sampling)
    closer = d < nearest                        # strict: an equally near smaller id keeps the voxel
    expanded[closer] = i
    nearest[closer] = d[closer]
  if max_distance is not None:
    far = edt > max_distance
    expanded[far] = seg[far]
  return expanded, edt


def unit_test_volumes():
  two = np.zeros((100, 80, 60), dtype=np.uint64)
  two[:40] = 1
  two[60:] = 2
  three = np.zeros((1, 100, 100), dtype=np.uint64)
  three[0, :20, :20] = 1
  three[0, :20:, -20:] = 2
  three[0, -20:, 40:60] = 3
  sparse = np.zeros((100, 80, 60), dtype=np.uint64)
  sparse[:40] = 1
  sparse[60, 0, 0] = 2
  sparse[61, 0, 0] = 2
  single = np.zeros((100, 80, 60), dtype=np.uint64)
  single[:40] = 1
  return two, three, sparse, single


def scattered_ids(n, rng):
  """n distinct uint64 ids: some below 2^32, some in [2^32, 2^63), some >= 2^63."""
  lo = rng.randint(1, 2**31, size=n // 3, dtype=np.int64).astype(np.uint64)
  mid = rng.randint(2**32, 2**62, size=n // 3, dtype=np.int64).astype(np.uint64) * np.uint64(2)
  hi = rng.randint(0, 2**62, size=n - 2 * (n // 3), dtype=np.int64).astype(np.uint64) + np.uint64(2**63)
  ids = np.concatenate([lo, mid, hi])
  assert np.unique(ids).size == n
  return ids[rng.permutation(n)]


def voronoi_cells(shape, seed, voxel_size_zyx, cell_volume, touching=False):
  """Voronoi cell ids (0 on the membranes unless touching) mapped onto scattered uint64 ids."""
  from ffn_b200.synthetic import voronoi_phantom
  _, cells = voronoi_phantom(shape, seed=seed, voxel_size_zyx=voxel_size_zyx, cell_volume=cell_volume,
                             return_cells=True)
  if touching:   # membrane voxels join the nearest cell, so that neighbouring cells touch
    idx = ndimage.distance_transform_edt(cells == 0, return_distances=False, return_indices=True)
    cells = cells[tuple(idx)]
  ncell = int(cells.max())
  lut = np.concatenate([[np.uint64(0)], scattered_ids(ncell, np.random.RandomState(seed + 1))])
  return lut[cells]


def cases():
  two, three, sparse, single = unit_test_volumes()
  iso = voronoi_cells((40, 64, 72), 21, (1.0, 1.0, 1.0), 4600.0)
  dusty = iso.copy()
  rng = np.random.RandomState(22)
  gaps = np.argwhere(iso == 0)
  for k, j in enumerate(rng.choice(len(gaps), 6, replace=False)):   # specks of 1 voxel in the gaps
    dusty[tuple(gaps[j])] = np.uint64(1000 + k)
  return [
      # name, seg, voxel size xyz, max_distance, box (start xyz, size xyz), optimize_sparse, threshold
      ('ut_two', two, (1, 1, 1), None, None, False, 0),
      ('ut_three', three, (1, 1, 1), None, None, False, 0),
      ('ut_three_md30', three, (1, 1, 1), 30.0, None, False, 0),
      ('ut_sparse', sparse, (1, 1, 1), None, None, False, 0),
      ('ut_sparse_opt0', sparse, (1, 1, 1), None, None, True, 0),
      ('ut_sparse_opt3', sparse, (1, 1, 1), None, None, True, 3),
      ('ut_single_opt0', single, (1, 1, 1), None, None, True, 0),
      ('voronoi_gaps', iso, (1, 1, 1), None, None, False, 0),
      ('voronoi_touch', voronoi_cells((40, 64, 72), 21, (1.0, 1.0, 1.0), 4600.0, touching=True), (1, 1, 1), None,
       None, False, 0),
      ('voronoi_dust', dusty, (1, 1, 1), None, None, True, 2),
      ('aniso_box', voronoi_cells((24, 64, 64), 23, (30.0, 8.0, 8.0), 2800.0), (8, 8, 30), 60.0,
       ((5, 7, 3), (50, 48, 18)), False, 0),
  ]


def main():
  os.environ.setdefault('PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION', 'python')
  mg.install_stubs()
  sys.modules['connectomics.common.bounding_box'].BoundingBox = Box
  sys.modules['connectomics.segmentation.labels'].watershed_expand = watershed_expand_definition
  sys.path.insert(0, mg.REF)
  from ffn.utils import decision_point as ref_dp

  out = {}
  names = []
  for name, seg, vs, md, box, opt, thr in cases():
    seg_in = seg.copy()
    work = seg.copy()
    res = ref_dp.find_decision_points(work, vs, max_distance=md, subvol_box=Box(*box) if box else None,
                                      optimize_sparse=opt, sparse_noise_threshold=thr)
    keys = list(res.keys())
    print(name, seg.shape, 'ids', np.unique(seg).size - 1, '->', len(keys), 'pairs',
          'dusted' if not np.array_equal(work, seg_in) else '', [(k, float(v[0]), v[1].tolist()) for k, v in
                                                                  list(res.items())[:2]])
    out[name + '_seg'] = seg_in
    out[name + '_seg_after'] = work
    out[name + '_voxel_size'] = np.asarray(vs, dtype=np.int64)
    out[name + '_max_distance'] = np.float64(np.nan if md is None else md)
    out[name + '_box'] = np.asarray(box[0] + box[1] if box else (), dtype=np.int64)
    out[name + '_optimize_sparse'] = np.bool_(opt)
    out[name + '_threshold'] = np.int64(thr)
    out[name + '_ids'] = np.asarray(keys, dtype=np.uint64).reshape(-1, 2)
    out[name + '_dist'] = np.asarray([res[k][0] for k in keys], dtype=np.float64)
    out[name + '_points'] = np.asarray([res[k][1] for k in keys], dtype=np.int64).reshape(-1, 3)
    names.append(name)
  out['cases'] = np.asarray(names)
  np.savez_compressed(os.path.join(HERE, 'decision_points_ref.npz'), **out)
  print('wrote decision_points_ref.npz')


if __name__ == '__main__':
  main()
