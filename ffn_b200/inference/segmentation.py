"""Label-volume helpers: saving results, connected-component clean-up and split consensus (ffn/inference/segmentation.py)."""

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


def clean_up(seg: np.ndarray, split_cc=True, connectivity=1, min_size=0, return_id_map=False, device=0):
  """Splits disconnected segments and clears dust, in place (ffn/inference/segmentation.py:89-118).

  See clean_up_and_count.

  Returns:
    None if not return_id_map, otherwise a dict mapping each output id to the original id at its first voxel
  """
  cc_to_orig, _ = clean_up_and_count(seg, split_cc, connectivity, min_size, compute_id_map=return_id_map,
                                     compute_counts=False, device=device)
  if return_id_map:
    return cc_to_orig


def clean_up_and_count(seg: np.ndarray, split_cc=True, connectivity=1, min_size=0, compute_id_map=True,
                       compute_counts=True, device=0):
  """Splits disconnected segments and clears dust, in place, and returns metadata (segmentation.py:121-178).

  With `split_cc`, every maximal set of voxels of one non-zero id that is connected under
  scipy.ndimage.generate_binary_structure(seg.ndim, connectivity) becomes one segment, numbered 1, 2, ... in C order
  of its first voxel (skimage.measure.label's numbering); this runs in libffn_b200 (ffn_clean_up), with no host
  fallback.  Then segments with fewer than `min_size` voxels become 0; the others keep their numbers, so ids have
  gaps.  Without `split_cc`, only the dust is cleared, on the host.

  Args:
    seg: uint64 segmentation with 1 to 3 dimensions; rewritten in place
    split_cc: whether to split disconnected segments
    connectivity: 1, 2 or 3 (6-, 18- or 26-connectivity in 3-D), at most seg.ndim
    min_size: segments with fewer voxels are cleared; <= 0: none are
    compute_id_map: whether to return {output id: original id at the id's first voxel} (None otherwise)
    compute_counts: whether to return {output id: voxel count} (None otherwise)
    device: CUDA device index (an H100)

  Returns:
    (id map, counts): dicts with np.uint64 keys, np.uint64 original ids and np.int64 counts.

  Raises:
    TypeError: if `seg` is not uint64
    ValueError: if split_cc and `connectivity` is not in [1, seg.ndim], or `seg` has more than 3 dimensions
    RuntimeError: if split_cc and `seg` has 2^31 or more voxels
  """
  if seg.dtype != np.uint64:
    raise TypeError('segmentation must be uint64, got %s' % seg.dtype)
  if not np.any(seg):
    if seg.size == 0:
      return ({} if compute_id_map else None, {} if compute_counts else None)
    zero = np.uint64(0)
    return ({zero: zero} if compute_id_map else None, {zero: np.int64(seg.size)} if compute_counts else None)

  if not split_cc:
    seg_orig = seg.copy() if compute_id_map else None
    if min_size > 0:
      clear_dust(seg, min_size)
    cc_to_orig, cc_to_count = None, None
    if compute_id_map or compute_counts:
      res = np.unique(seg.ravel(), return_index=compute_id_map, return_counts=compute_counts)
      if compute_id_map:
        cc_to_orig = dict(zip(res[0], seg_orig.ravel()[res[1]]))
      if compute_counts:
        cc_to_count = dict(zip(res[0], res[-1]))
    return cc_to_orig, cc_to_count

  if seg.ndim > 3:
    raise ValueError('connected components of %d-D segmentations are not supported' % seg.ndim)
  if not 1 <= connectivity <= seg.ndim:
    raise ValueError('connectivity for a %d-D segmentation must be in [1, %d], got %r' % (
        seg.ndim, seg.ndim, connectivity))
  if seg.size >= 2**31:
    raise RuntimeError('connected components support volumes of fewer than 2^31 voxels')
  from ffn_b200 import _lib
  # Counts are integers below 2^31: count < min_size is count < ceil(min_size), which fits in an int64.
  ms = int(min(max(np.ceil(min_size), -2.0**62), 2.0**62))
  desc = _lib.CleanUpDesc(_lib.i3((1,) * (3 - seg.ndim) + seg.shape), int(connectivity), ms)
  work = seg if seg.flags.c_contiguous else np.ascontiguousarray(seg)
  table = compute_id_map or compute_counts
  # Room for components of 64 voxels on average: a larger table repeats the whole call, upload included.
  cap = min(seg.size + 1, max(4096, seg.size // 64)) if table else 0
  lib = _lib.load()
  n_ids = _lib.C.c_int64(0)
  while True:
    ids, orig, counts = (np.empty(cap, np.uint64), np.empty(cap, np.uint64), np.empty(cap, np.int64))
    _lib.check(lib.ffn_clean_up(int(device), _lib.C.byref(desc), _lib.ptr(work),
                                *((_lib.ptr(ids), _lib.ptr(orig), _lib.ptr(counts)) if table else (None,) * 3),
                                cap, _lib.C.byref(n_ids)))
    if n_ids.value <= cap:
      break
    cap = n_ids.value   # the table did not fit and nothing was written: again, with room for every row
  if work is not seg:
    seg[...] = work
  k = n_ids.value
  return (dict(zip(ids[:k], orig[:k])) if compute_id_map else None,
          dict(zip(ids[:k], counts[:k])) if compute_counts else None)
