"""Numpy restatement of compute_partitions (compute_partitions.py:115-204), with tuple indexing.

Each label's summed-volume table covers only its bounding box clipped to the VALID centres and grown by the LOM
radius, so the work is the sum of those boxes instead of labels x voxels.  The exclusion spheres use the reference's
own numpy expression; the mask is any() over the LOM box, from a summed-volume table.  It shares no code with the
device path.
"""

import numpy as np


def clear_dust(seg, min_size):
  """Zeroes non-zero ids with fewer than `min_size` voxels, in place (segmentation.py:21-63)."""
  if seg.size == 0 or min_size <= 0:
    return seg
  ids, sizes = np.unique(seg, return_counts=True)
  small = ids[(sizes < min_size) & (ids != 0)]
  if small.size:
    seg[np.isin(seg, small)] = 0
  return seg


def _window_sums(val, r):
  """VALID sums of `val` over (2r + 1) boxes (r in z, y, x), exact in int64."""
  svt = np.pad(val.astype(np.int64).cumsum(0).cumsum(1).cumsum(2), [[1, 0], [1, 0], [1, 0]])
  d = [2 * x + 1 for x in r]
  hi = [slice(di, None) for di in d]
  lo = [slice(None, svt.shape[a] - d[a]) for a in range(3)]
  s = 0
  for bits in range(8):
    sel = tuple(lo[a] if bits >> (2 - a) & 1 else hi[a] for a in range(3))
    s = s + (-1) ** bin(bits).count('1') * svt[sel]
  return s


def compute_partitions(seg, thresholds, lom_radius, id_whitelist=None, exclusion_regions=None, mask=None,
                       min_size=10000):
  """`mask`: the boolean volume of build_mask(mask_configs.masks, (0, 0, 0), seg.shape), or None.

  Returns (corner, uint8 partitions); `seg` is cleared of dust in place."""
  clear_dust(seg, min_size)
  corner = np.array(lom_radius)
  r = [int(x) for x in corner[::-1]]
  out = np.zeros([max(0, s - 2 * x) for s, x in zip(seg.shape, r)], np.uint8)

  if exclusion_regions is not None:
    hz, hy, hx = np.mgrid[:out.shape[0], :out.shape[1], :out.shape[2]]
    hz += corner[2]
    hy += corner[1]
    hx += corner[0]
    for x, y, z, rad in exclusion_regions:
      out[(hx - x)**2 + (hy - y)**2 + (hz - z)**2 <= rad**2] = 255

  labels = set(np.unique(seg).tolist())
  if id_whitelist is not None:
    labels &= set(id_whitelist)
  labels.discard(0)

  if mask is not None and out.size:
    out[_window_sums(mask, r) >= 1] = 255

  if labels and len(thresholds) == 0:
    raise IndexError('list index out of range')
  if labels and len(thresholds) + 1 > 255:
    raise OverflowError('Python integer %d out of bounds for uint8' % (len(thresholds) + 1))
  fov = np.prod([2 * x + 1 for x in r])
  th = [float(t) for t in thresholds]
  for lab in sorted(labels):
    obj = seg == lab
    where = np.nonzero(obj)
    lo = [max(int(w.min()), x) - x for w, x in zip(where, r)]
    hi = [min(int(w.max()) + 1, s - x) + x for w, s, x in zip(where, seg.shape, r)]
    if any(h - l <= 2 * x for l, h, x in zip(lo, hi, r)):
      continue   # no voxel of this label in the VALID region
    box = tuple(slice(l, h) for l, h in zip(lo, hi))
    frac = _window_sums(obj[box], r) / fov
    inner = obj[box][tuple(slice(x, obj[box].shape[a] - x) for a, x in enumerate(r))]
    q = np.full(frac.shape, len(th) + 1, np.uint8)
    done = np.zeros(frac.shape, bool)
    for i, t in enumerate(th):
      hit = ~done & (frac < t)
      q[hit] = i + 1
      done |= hit
    dst = out[tuple(slice(l, h - 2 * x) for l, h, x in zip(lo, hi, r))]
    sel = inner & (dst == 0)
    dst[sel] = q[sel]
  return corner, out
