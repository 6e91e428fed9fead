"""Oracle: the PolicyPeaks2d / PolicyFillEmptySpace / PolicyMaxPeaks seed lists on the CPU (TEST INFRASTRUCTURE —
only tests/ may import this; the product never does).

Restates ffn/inference/seed.py:202-352 together with `_find_peaks` (:133-139), `get_exclusion_mask` (:118-130) and
the border filter of `BaseSeedPolicy.__next__` (:81-88), independently of `ffn_b200` (nothing from the product
package is imported here; the Sobel / gaussian edge map is the one of oracle/seed_peaks.py).

PINNED against the reference's own, unmodified policies (tests/golden/make_golden_peak_policies.py ->
peak_policies_ref.npz: seed lists equal, order included), except for the two un-vendored third-party calls, which
that fixture injects by the same published definitions as oracle/seed_peaks.py describes (exact EDT; peak_local_max
with threshold_abs=None meaning the minimum and exclude_border=min_distance on every axis of the array).

Where a slice (PolicyPeaks2d) or the canvas (PolicyFillEmptySpace) has no background voxel, the distance is nowhere
finite and the reference's result depends on the un-vendored `edt`; that case is DEFINED here as "no seeds" and is
not pinned.
"""

from __future__ import annotations

import numpy as np
from scipy import ndimage

from .seed_peaks import edge_map


def peak_local_max_full(values: np.ndarray, min_distance: int, threshold_abs=None, threshold_rel=None) -> np.ndarray:
  """Documented skimage semantics with the full threshold set; rows in C order.  threshold_abs=None means the
  minimum (skimage), threshold_rel=None means no relative threshold; non-finite values are never peaks."""
  values = np.asarray(values, dtype=np.float64)
  ok = np.isfinite(values)
  if not ok.any():
    return np.zeros((0, values.ndim), dtype=np.int64)
  threshold = float(np.min(values[ok])) if threshold_abs is None else float(threshold_abs)
  if threshold_rel is not None:
    threshold = max(threshold, float(threshold_rel) * float(np.max(values[ok])))
  box = ndimage.maximum_filter(values, size=2 * min_distance + 1, mode='nearest')
  keep = ok & (values == box) & (values > threshold)
  lo = min_distance
  for axis, s in enumerate(values.shape):                            # exclude_border=min_distance on every axis
    idx = np.arange(s)
    inside = (idx >= lo) & (idx < s - lo)
    keep &= inside.reshape([-1 if a == axis else 1 for a in range(values.ndim)])
  return np.argwhere(keep)


def _border_filter(coords, shape, margin_zyx):
  if margin_zyx is None or not coords.size:
    return coords
  m = np.asarray(margin_zyx)[None]
  return coords[np.all((coords - m >= 0) & (coords + m < np.asarray(shape)[None]), axis=1)]


def policy_peaks_2d(image_f32: np.ndarray, mask=None, min_distance=7, threshold_abs=2.5, sort_cmp='ascending',
                    margin_zyx=None) -> np.ndarray:
  """The seed list PolicyPeaks2d yields, in order: [N, 3] int64 (z, y, x)."""
  image_f32 = np.asarray(image_f32)
  noise = np.random.RandomState(seed=42).rand(*image_f32.shape[1:])   # one plane, the same for every slice
  rows = []
  for z in range(image_f32.shape[0]):
    filt_edges = edge_map(image_f32[z])                                # 2-D Sobel + 2-D gaussian threshold
    if mask is not None:
      filt_edges[np.asarray(mask[z]).astype(bool)] = True
    if not filt_edges.any():                                           # no finite distance: no seeds (unpinned)
      continue
    dt = ndimage.distance_transform_edt(~filt_edges).astype(np.float32)
    for y, x in peak_local_max_full(dt + noise * 1e-4, min_distance, threshold_abs, 0):
      rows.append((z, int(y), int(x)))
  coords = np.array(sorted(rows, reverse=sort_cmp.strip().lower().startswith('de')), dtype=np.int64).reshape(-1, 3)
  return _border_filter(coords, image_f32.shape, margin_zyx)


def policy_fill_empty_space(segmentation: np.ndarray, margin_zyx=None) -> np.ndarray:
  """The seed list PolicyFillEmptySpace yields: peaks of the EDT of the unlabelled voxels."""
  seg = np.asarray(segmentation)
  if np.all(seg == 0):                                                 # no finite distance: no seeds (unpinned)
    return np.zeros((0, 3), dtype=np.int64)
  dt = ndimage.distance_transform_edt(seg == 0).astype(np.float32)
  noise = np.random.RandomState(seed=42).rand(*seg.shape)
  idx = peak_local_max_full(dt + noise * 1e-4, 2, 0.5, 0)
  coords = np.array(sorted(tuple(int(v) for v in r) for r in idx), dtype=np.int64).reshape(-1, 3)
  return _border_filter(coords, seg.shape, margin_zyx)


def policy_max_peaks(image_f32: np.ndarray, segmentation=None, mask=None, seed_mask=None, min_distance=3,
                     threshold_abs=0, threshold_rel=0, margin_zyx=None) -> np.ndarray:
  """The seed list PolicyMaxPeaks yields: intensity peaks with labels / mask / seed mask set to 0."""
  img = np.array(image_f32, dtype=np.float32)
  excl = np.zeros(img.shape, dtype=bool) if segmentation is None else (np.asarray(segmentation) > 0)
  for m in (mask, seed_mask):
    if m is not None:
      excl |= np.asarray(m).astype(bool)
  img[excl] = 0
  noise = np.random.RandomState(seed=42).rand(*img.shape)
  idx = peak_local_max_full(img + noise * 1e-4, min_distance, threshold_abs, threshold_rel)
  coords = np.array(sorted(tuple(int(v) for v in r) for r in idx), dtype=np.int64).reshape(-1, 3)
  return _border_filter(coords, img.shape, margin_zyx)
