"""Decision points of a segmentation on the device: find_decision_points (ffn/utils/decision_point.py:27-145).

A decision point of two objects is where they come closest once every empty voxel has taken the id of the
nearest object.  Resegmentation (ffn_b200/inference/resegmentation.py) starts from these (id_a, id_b, point)
triples.  The computation runs in libffn_b200 (ffn_decision_points); there is no host fallback.
"""

from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np

from ffn_b200 import _lib

# Output slots of the first call; a larger result is fetched again with room for all of it.
_INITIAL_CAP = 4096


def _voxel_size(voxel_size) -> tuple:
  vs = tuple(voxel_size)
  if len(vs) != 3:
    raise ValueError('voxel_size must have 3 components (x, y, z), got %r' % (voxel_size,))
  out = []
  for v in vs:
    try:
      iv = int(v)
      ok = iv == v and 0 < iv < 2**31
    except (TypeError, ValueError, OverflowError):
      ok = False
    if not ok:
      raise ValueError('voxel sizes must be positive integers below 2^31, got %r' % (voxel_size,))
    out.append(iv)
  return tuple(out)


def _box(subvol_box, shape):
  """(start, size) in (z, y, x) from a box's slices; the whole volume when there is no box."""
  if subvol_box is None:
    return (0, 0, 0), tuple(shape)
  slices = subvol_box.to_slice3d() if hasattr(subvol_box, 'to_slice3d') else subvol_box.to_slice()
  if len(slices) != 3:
    raise ValueError('subvol_box must select 3 axes, got %r' % (slices,))
  start, size = [], []
  for sl, n in zip(slices, shape):
    lo, hi = sl.start, sl.stop
    if sl.step not in (None, 1) or lo is None or hi is None or not 0 <= int(lo) <= int(hi) <= n:
      raise ValueError('subvol_box %r lies outside the volume of shape %r' % (subvol_box, tuple(shape)))
    start.append(int(lo))
    size.append(int(hi) - int(lo))
  return tuple(start), tuple(size)


def find_decision_points(
    seg: np.ndarray,
    voxel_size: Sequence[float],
    max_distance: Optional[float] = None,
    subvol_box=None,
    optimize_sparse: bool = False,
    sparse_noise_threshold: int = 0,
    device: int = 0,
) -> dict:
  """Identifies decision points in a segmentation subvolume.

  Args:
    seg: 3d array of non-negative integer segment ids (z, y, x)
    voxel_size: (x, y, z) physical voxel size; positive integers
    max_distance: maximum distance between a segment and the decision point (units of voxel_size); None: no limit
    subvol_box: BoundingBox (or any box with `to_slice3d`) within which to search for decision points; the whole
      volume is always used for the distance transform
    optimize_sparse: if True and sparse_noise_threshold > 0, objects with fewer voxels than the threshold are first
      cleared from `seg`, in place
    sparse_noise_threshold: see optimize_sparse
    device: CUDA device index (an H100)

  Returns:
    dict from (id_a, id_b), id_a < id_b, in ascending order, to (distance, np.int64 [x, y, z] point relative to the
    box)
  """
  if not isinstance(seg, np.ndarray) or seg.ndim != 3:
    raise ValueError('seg must be a 3d numpy array')
  if not np.issubdtype(seg.dtype, np.integer):
    raise ValueError('seg must hold integer ids, got dtype %s' % seg.dtype)
  if seg.size and np.issubdtype(seg.dtype, np.signedinteger) and seg.min() < 0:
    raise ValueError('seg must not contain negative ids')
  vs = _voxel_size(voxel_size)
  start, size = _box(subvol_box, seg.shape)
  if seg.size == 0:
    return {}
  threshold = int(sparse_noise_threshold) if optimize_sparse else 0

  desc = _lib.DecisionPointDesc()
  desc.shape_zyx[:] = seg.shape
  desc.voxel_size_xyz[:] = vs
  desc.use_max_distance = int(max_distance is not None)
  desc.max_distance = float(max_distance) if max_distance is not None else 0.0
  desc.box_start_zyx[:] = start
  desc.box_size_zyx[:] = size
  desc.dust_threshold = max(threshold, 0)
  labels = np.array(seg, dtype=np.uint64, order='C', copy=True)
  lib = _lib.load()
  cap = _INITIAL_CAP
  while True:
    out = np.zeros(cap, dtype=_lib.DECISION_POINT_DTYPE)
    n = C.c_int64(0)
    _lib.check(lib.ffn_decision_points(int(device), C.byref(desc), _lib.ptr(labels), _lib.ptr(out), cap, C.byref(n)))
    if n.value <= cap:
      break
    cap = n.value
  if threshold > 0:
    seg[labels == 0] = 0
  return {(int(p['id_a']), int(p['id_b'])): (np.float64(p['dist']), p['point_xyz'].copy())
          for p in out[:n.value]}
