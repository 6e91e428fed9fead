"""Numpy restatement of build_coordinates' main (build_coordinates.py:61-112), with the reference's own 2-d calls.

Partitions are collected per value in first-seen order (volume by volume, ascending within a volume), each one's
(volume, flat index) rows are permuted and repeated cyclically to the largest partition's size with
np.random.permutation and np.resize on (n, 2) int64 arrays, and the concatenation is shuffled with np.random.shuffle,
all on numpy's global RandomState.  It shares no code with the device path.
"""

import numpy as np

IGNORE_PARTITION = 255


def coordinate_rows(volumes, margin_zyx):
  """Shuffled (n, 2) int64 rows (volume index, flat crop index) and the crop shapes; ValueError when no crop holds a
  partition other than 255."""
  mz, my, mx = [int(m) for m in margin_zyx]
  indices = {}   # partition -> [(n, 2) rows], in first-seen order
  shapes = []
  for i, vol in enumerate(volumes):
    crop = np.asarray(vol)[mz:-mz, my:-my, mx:-mx]
    shapes.append(crop.shape)
    for val in np.unique(crop):
      if val == IGNORE_PARTITION:
        continue
      flat = np.flatnonzero(crop == val).astype(np.int64)
      indices.setdefault(int(val), []).append(np.stack([np.full(flat.size, i, np.int64), flat], axis=1))
  max_count = max(sum(len(r) for r in v) for v in indices.values())
  rows = np.concatenate([np.resize(np.random.permutation(np.concatenate(v)), (max_count, 2))
                         for v in indices.values()], axis=0)
  np.random.shuffle(rows)
  return rows, shapes


def build_coordinates(volumes, margin_zyx):
  """(centers (n, 3) int64 as [x, y, z], volume index (n,) int64) of every record, in file order."""
  mz, my, mx = [int(m) for m in margin_zyx]
  rows, shapes = coordinate_rows(volumes, margin_zyx)
  centers = np.empty((len(rows), 3), np.int64)
  for i, shape in enumerate(shapes):
    sel = rows[:, 0] == i
    if sel.any():
      z, y, x = np.unravel_index(rows[sel, 1], shape)
      centers[sel] = np.stack([mx + x, my + y, mz + z], axis=1)
  return centers, rows[:, 0].copy()
