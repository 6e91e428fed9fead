"""Label-volume helpers: saving results and split consensus (subset of ffn/inference/segmentation.py)."""

import numpy as np


def reduce_id_bits(segmentation: np.ndarray) -> np.ndarray:
  """Smallest unsigned dtype holding every id (ffn/inference/segmentation.py:66-86)."""
  max_id = segmentation.max() if segmentation.size else 0
  for dt in (np.uint8, np.uint16, np.uint32):
    if max_id <= np.iinfo(dt).max:
      return segmentation.astype(dt)
  return segmentation


def clear_dust(data: np.ndarray, min_size: int = 10) -> np.ndarray:
  """Zeroes segments smaller than `min_size` voxels, in place (segmentation.py:21-63)."""
  ids, sizes = np.unique(data, return_counts=True)
  small = ids[sizes < min_size]
  if small.size:
    data[np.isin(data, small)] = 0
  return data


def split_segmentation_by_intersection(a: np.ndarray, b: np.ndarray, min_size: int, device: int = 0) -> None:
  """Splits `a` by its intersection with `b`, in place (ffn/inference/segmentation.py:181-290).

  Every overlapping (id_a, id_b) pair of voxels becomes one segment.  It keeps id_a when id_b is id_a's largest
  overlap (the smallest id_b on equal counts); the other pairs get new ids max(a) + 1, max(a) + 2, ... in (id_b, id_a)
  order.  Pairs smaller than `min_size` voxels and pairs with id_a == 0 become 0; (id_a, 0) pairs are kept.  `b` is
  not changed.  Runs in libffn_b200 (ffn_split_intersection); there is no host fallback.

  Args:
    a: first segmentation, uint64; rewritten in place
    b: second segmentation, uint64, same shape
    min_size: minimum size in voxels of a segment created by the intersection
    device: CUDA device index (an H100)

  Raises:
    ValueError: if a.shape != b.shape or `a` is empty
    TypeError: if a or b is not uint64
    RuntimeError: if `a` has 2^31 or more voxels, or max(a) plus the number of new ids does not fit in 64 bits
  """
  from ffn_b200 import _lib
  if a.shape != b.shape:
    raise ValueError('segmentations differ in shape: %r, %r' % (a.shape, b.shape))
  if a.dtype != np.uint64:
    raise TypeError('segmentation must be uint64, got %s' % a.dtype)
  if a.size == 0:
    raise ValueError('zero-size segmentation')
  if b.dtype != np.uint64:
    raise TypeError('segmentation must be uint64, got %s' % b.dtype)
  # Counts are integers below 2^31: count < min_size is count < ceil(min_size), which fits in an int64.
  ms = int(min(max(np.ceil(min_size), -2.0**62), 2.0**62))
  work = a if a.flags.c_contiguous else np.ascontiguousarray(a)
  bc = np.ascontiguousarray(b)
  lib = _lib.load()
  _lib.check(lib.ffn_split_intersection(int(device), work.size, _lib.ptr(work), _lib.ptr(bc), ms))
  if work is not a:
    a[...] = work
