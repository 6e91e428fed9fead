"""Host oracle of find_decision_points (ffn/utils/decision_point.py:27-145), restated in numpy from its definition.

  1. optimize_sparse with a threshold > 0: ids with fewer voxels than the threshold become 0, in place.
  2. Nearest-id expansion: every empty voxel takes the id of the nearest labelled voxel (squared physical distance
     with sampling = voxel_size[::-1]; the smallest id on ties); edt = the distance to it.  Where
     edt > max_distance the expansion keeps the input (0).  Here one exact feature transform per id
     (scipy.ndimage.distance_transform_edt) gives that id's integer squared distance, so ties are found exactly.
  3. Within the box, for the offsets of itertools.product((0, -1), (0, -1), (0, -1)) without (0, 0, 0): rows
     (a-voxel, b-voxel = a-voxel + |offset|) with both ids > 0 and different; dist = (edt_a + edt_b) / 2.
  4. Per pair (a, b), a < b: the rows at the minimal dist; their centroid = int64 coordinate sum / count; the point
     is the row with the least ((x-mx)^2 + (y-my)^2) + (z-mz)^2, the first in (offset, raster) order on ties.
"""

from __future__ import annotations

import itertools

import numpy as np
from scipy import ndimage


def clear_dust(seg: np.ndarray, min_size: int) -> None:
  if min_size <= 0 or seg.size == 0:
    return
  ids, counts = np.unique(seg, return_counts=True)
  small = ids[(counts < min_size) & (ids != 0)]
  if small.size:
    seg[np.isin(seg, small)] = 0


def nearest_id(seg: np.ndarray, voxel_size_xyz):
  """(expanded ids, integer squared distance D) of every voxel; D = -1 where no labelled voxel exists."""
  w = np.asarray(voxel_size_xyz, dtype=np.int64)[::-1]
  expanded = np.zeros(seg.shape, dtype=np.uint64)
  best = np.full(seg.shape, -1, dtype=np.int64)
  if not (seg == 0).any():   # nothing to expand
    return seg.astype(np.uint64), np.zeros(seg.shape, dtype=np.int64)
  grid = np.indices(seg.shape, dtype=np.int64)
  for i in np.unique(seg[seg != 0]):   # ascending: a later id only wins when strictly nearer
    feat = ndimage.distance_transform_edt(seg != i, sampling=w.astype(np.float64), return_distances=False,
                                          return_indices=True)
    d2 = np.zeros(seg.shape, dtype=np.int64)
    for a in range(3):
      d2 += ((feat[a].astype(np.int64) - grid[a]) * w[a]) ** 2
    take = (best < 0) | (d2 < best)
    expanded[take] = i
    best[take] = d2[take]
  return expanded, best


def watershed_expand(seg: np.ndarray, voxel_size_xyz, max_distance=None):
  expanded, d2 = nearest_id(seg, voxel_size_xyz)
  edt = np.sqrt(np.maximum(d2, 0).astype(np.float64))
  if max_distance is not None:
    far = edt > max_distance
    expanded[far] = seg[far]
  return expanded, edt


def find_decision_points(seg, voxel_size, max_distance=None, subvol_box=None, optimize_sparse=False,
                         sparse_noise_threshold=0):
  if optimize_sparse:
    clear_dust(seg, int(sparse_noise_threshold))
  expanded, edt = watershed_expand(seg, voxel_size, max_distance)
  if subvol_box is not None:
    sl = subvol_box.to_slice3d() if hasattr(subvol_box, 'to_slice3d') else subvol_box.to_slice()
    expanded, edt = expanded[sl], edt[sl]
  return points_of_expansion(expanded, edt)


def points_of_expansion(expanded, edt):
  """Steps 3 and 4 on an expanded segmentation and its distances (already cut to the box)."""
  cols = {k: [] for k in ('a', 'b', 'dist', 'x', 'y', 'z')}
  shape = expanded.shape
  for off in itertools.product((0, 1), (0, 1), (0, 1)):
    if off == (0, 0, 0):
      continue
    lo = tuple(slice(0, n - o) for n, o in zip(shape, off))
    hi = tuple(slice(o, n) for n, o in zip(shape, off))
    ea, eb = expanded[lo], expanded[hi]
    t = (ea > 0) & (eb > 0) & (ea != eb)
    z, y, x = np.nonzero(t)
    cols['a'].append(np.minimum(ea[t], eb[t]))
    cols['b'].append(np.maximum(ea[t], eb[t]))
    cols['dist'].append((edt[lo][t] + edt[hi][t]) / 2)
    for k, v in (('x', x), ('y', y), ('z', z)):
      cols[k].append(v.astype(np.int64))
  a, b, dist, x, y, z = (np.concatenate(cols[k]) for k in ('a', 'b', 'dist', 'x', 'y', 'z'))
  if a.size == 0:
    return {}

  order = np.lexsort((b, a))   # stable: rows of a pair stay in (offset, raster) order
  a, b, dist, x, y, z = a[order], b[order], dist[order], x[order], y[order], z[order]
  starts = np.flatnonzero(np.r_[True, (a[1:] != a[:-1]) | (b[1:] != b[:-1])])
  ends = np.r_[starts[1:], a.size]
  ret = {}
  for s, e in zip(starts, ends):
    d = dist[s:e]
    m = d == d.min()
    px, py, pz = x[s:e][m], y[s:e][m], z[s:e][m]
    cnt = px.size
    mx, my, mz = px.sum() / cnt, py.sum() / cnt, pz.sum() / cnt
    c2 = ((px - mx) ** 2 + (py - my) ** 2) + (pz - mz) ** 2
    k = int(np.argmin(c2))
    ret[(int(a[s]), int(b[s]))] = (np.float64(d.min()), np.array([px[k], py[k], pz[k]], dtype=np.int64))
  return ret
