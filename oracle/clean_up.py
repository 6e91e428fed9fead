"""Numpy / scipy restatement of connected-component clean-up (ffn/inference/segmentation.py:89-178).

A component is a maximal set of voxels of one non-zero id connected under
scipy.ndimage.generate_binary_structure(ndim, connectivity); components are numbered 1, 2, ... in C order of their
first voxel, and 0 stays 0 (what skimage.measure.label(seg, connectivity=c, background=0) returns).  Each id is
labelled inside its ndimage.find_objects box, so the work is the sum of the box volumes, not ids x voxels.  Dust and
the id map / counts then follow the reference's clean_up_and_count step by step.  It shares no code with the device
path.
"""

import numpy as np
from scipy import ndimage


def split_disconnected_components(seg, connectivity=1):
  """The components of `seg` (any integer dtype), as an int64 array of the same shape."""
  if not 1 <= connectivity <= seg.ndim:
    raise ValueError('connectivity must be in [1, %d], got %r' % (seg.ndim, connectivity))
  structure = ndimage.generate_binary_structure(seg.ndim, connectivity)
  ids, compact = np.unique(seg, return_inverse=True)
  compact = compact.reshape(seg.shape)
  if ids[0] != 0:
    compact = compact + 1   # find_objects treats 0 as background
  first = np.full(seg.shape, -1, np.int64)   # per foreground voxel: the flat index of its component's first voxel
  for k, box in enumerate(ndimage.find_objects(compact), start=1):
    if box is None:
      continue
    mask = compact[box] == k
    lab, _ = ndimage.label(mask, structure)
    # C order inside a box is C order in the volume, so a component's first voxel in the box is its first voxel
    comp_ids, at = np.unique(lab.ravel(), return_index=True)
    first_of = np.zeros(comp_ids.max() + 1, np.int64)
    local = np.unravel_index(at, mask.shape)
    first_of[comp_ids] = np.ravel_multi_index(tuple(l + b.start for l, b in zip(local, box)), seg.shape)
    first[box][mask] = first_of[lab[mask]]
  out = np.zeros(seg.shape, np.int64)
  fg = first >= 0
  out[fg] = np.unique(first[fg], return_inverse=True)[1].ravel() + 1
  return out


def clear_dust(seg, min_size):
  ids, sizes = np.unique(seg, return_counts=True)
  small = ids[(sizes < min_size) & (ids != 0)]
  if small.size:
    seg[np.isin(seg, small)] = 0
  return seg


def clean_up_and_count(seg, split_cc=True, connectivity=1, min_size=0, compute_id_map=True, compute_counts=True):
  """`seg` is modified in place; returns (id map, counts) as the reference does."""
  if not np.any(seg):
    if seg.size == 0:
      return ({} if compute_id_map else None, {} if compute_counts else None)
    zero = seg.dtype.type(0)
    return ({zero: zero} if compute_id_map else None, {zero: np.int64(seg.size)} if compute_counts else None)
  seg_orig = seg.copy()
  if split_cc:
    seg[...] = split_disconnected_components(seg, connectivity)
  if min_size > 0:
    clear_dust(seg, min_size)
  cc_to_orig, cc_to_count = None, None
  if compute_id_map or compute_counts:
    res = np.unique(seg.ravel(), return_index=True, return_counts=True)
    if compute_id_map:
      cc_to_orig = dict(zip(res[0], seg_orig.ravel()[res[1]]))
    if compute_counts:
      cc_to_count = dict(zip(res[0], res[2]))
  return cc_to_orig, cc_to_count


def clean_up(seg, split_cc=True, connectivity=1, min_size=0, return_id_map=False):
  cc_to_orig, _ = clean_up_and_count(seg, split_cc, connectivity, min_size, compute_id_map=return_id_map,
                                     compute_counts=False)
  if return_id_map:
    return cc_to_orig
