"""numpy / scipy restatement of resegmentation_analysis.evaluate_{pair,endpoint}_resegmentation (tests only).

Follows ffn/inference/resegmentation_analysis.py:97-260 step by step on the host: scipy's distance_transform_edt for
the four distance maps, numpy for the masks and counts, np.unique for ComputeOverlapCounts.  The device path
(ffn_b200/inference/resegmentation_analysis.py) is compared against this.
"""

import re

import numpy as np
from scipy import ndimage

from ffn_b200.inference import resegmentation_pb2, storage


class InvalidBaseSegmentatonError(Exception):
  pass


class IncompleteResegmentationError(Exception):
  pass


def parse_resegmentation_filename(filename):
  return tuple(int(t) for t in re.search(r'(\d+)-(\d+)_at_(\d+)_(\d+)_(\d+)', filename).groups())


def _crop(seg_volume, z, y, x, r):
  crop = np.asarray(seg_volume[0, (z - r[0]):(z + r[0] + 1), (y - r[1]):(y + r[1] + 1), (x - r[2]):(x + r[2] + 1)])
  return crop[0, ...] if crop.ndim == 4 else crop


def _load(filename):
  return np.load(filename, allow_pickle=True)


def _segment_result(reseg, dels, moves, delta, analysis_r, seg1, seg2, sampling, result):
  result.max_edt = float(ndimage.distance_transform_edt(reseg, sampling=sampling).max())
  if moves.size > 0:
    lo, hi = np.array(delta), np.array(delta) + 2 * np.array(analysis_r)
    inside = np.all((moves >= lo[np.newaxis]) & (moves <= hi[np.newaxis]), axis=1)
    result.deleted_voxels = int(np.sum(dels[inside]))
  result.num_voxels = int(np.sum(reseg))
  result.segment_a_consistency = float(np.sum(reseg[seg1])) / np.sum(seg1)
  result.segment_b_consistency = float(np.sum(reseg[seg2])) / np.sum(seg2)


def evaluate_pair_resegmentation(filename, seg_volume, resegmentation_radius, analysis_radius, voxel_size,
                                 threshold=0.5):
  id1, id2, x, y, z = parse_resegmentation_filename(filename)
  result = resegmentation_pb2.PairResegmentationResult()
  result.id_a, result.id_b = id1, id2
  result.point.x, result.point.y, result.point.z = x, y, z
  sr = result.segmentation_radius
  sr.z, sr.y, sr.x = resegmentation_radius
  data = _load(filename)
  prob = np.nan_to_num(storage.dequantize_probability(data['probs']))
  dels, moves, start_points = data['deletes'], data['histories'], data['start_points']
  if prob.shape[0] != 2:
    raise IncompleteResegmentationError()
  corner = np.array([x - sr.x, y - sr.y, z - sr.z])
  oa, ob = result.eval.from_a.origin, result.eval.from_b.origin
  oa.x, oa.y, oa.z = np.array(start_points[0][-1], dtype=int) + corner
  ob.x, ob.y, ob.z = np.array(start_points[1][-1], dtype=int) + corner
  ar = np.array(analysis_radius)
  result.eval.radius.z, result.eval.radius.y, result.eval.radius.x = ar
  seg = _crop(seg_volume, z, y, x, ar)
  seg1, seg2 = seg == id1, seg == id2
  result.eval.num_voxels_a = int(np.sum(seg1))
  result.eval.num_voxels_b = int(np.sum(seg2))
  if result.eval.num_voxels_a == 0 or result.eval.num_voxels_b == 0:
    raise InvalidBaseSegmentatonError()
  result.eval.max_edt_a = float(ndimage.distance_transform_edt(seg1, sampling=voxel_size).max())
  result.eval.max_edt_b = float(ndimage.distance_transform_edt(seg2, sampling=voxel_size).max())
  delta = np.array(resegmentation_radius) - ar
  reseg = prob[:, delta[0]:(delta[0] + 2 * ar[0] + 1), delta[1]:(delta[1] + 2 * ar[1] + 1),
               delta[2]:(delta[2] + 2 * ar[2] + 1)] >= threshold
  with np.errstate(invalid='ignore', divide='ignore'):
    result.eval.iou = np.sum(reseg[0] & reseg[1]) / float(np.sum(reseg[0] | reseg[1]))
  _segment_result(reseg[0], dels[0], moves[0], delta, ar, seg1, seg2, voxel_size, result.eval.from_a)
  _segment_result(reseg[1], dels[1], moves[1], delta, ar, seg1, seg2, voxel_size, result.eval.from_b)
  return result


def evaluate_endpoint_resegmentation(filename, seg_volume, resegmentation_radius, threshold=0.5):
  id1, _, x, y, z = parse_resegmentation_filename(filename)
  result = resegmentation_pb2.EndpointResegmentationResult()
  result.id = id1
  result.start.x, result.start.y, result.start.z = x, y, z
  sr = result.segmentation_radius
  sr.z, sr.y, sr.x = resegmentation_radius
  prob = np.nan_to_num(storage.dequantize_probability(_load(filename)['probs']))
  orig = _crop(seg_volume, z, y, x, (sr.z, sr.y, sr.x))
  if not np.any(orig == id1):
    raise InvalidBaseSegmentatonError()
  new = prob[0] >= threshold
  result.num_voxels = int(np.sum(new))
  ids, totals = np.unique(orig, return_counts=True)
  inside, counts = np.unique(orig[new], return_counts=True)
  for old_u, v in zip(inside, counts):
    old = int(old_u)
    result.overlaps[old].num_overlapping = int(v)
    result.overlaps[old].num_original = int(totals[np.searchsorted(ids, old_u)])   # uint64 key: no float rounding
    if old == id1:
      result.source.CopyFrom(result.overlaps[old])
  return result


def _grow(mask, steps):
  out = mask.copy()
  for _ in range(steps):
    for axis in range(3):
      lo, hi = [slice(None)] * 3, [slice(None)] * 3
      lo[axis], hi[axis] = slice(1, None), slice(None, -1)
      out[tuple(lo)] |= out[tuple(hi)].copy()
      out[tuple(hi)] |= out[tuple(lo)].copy()
  return out


def write_synthetic_results(seg, points, radius_zyx, directory, seed=0):
  """A result file of process_point's layout per (id_a, id_b, point_xyz) whose resegmentation box fits into `seg`
  ([Z, Y, X]): object k is its original segment, grown by 0-2 voxels, half of the time merged with the other one,
  with unvisited voxels; 1-3 attempts and 3-12 FoV moves per object.  Returns the paths written."""
  import os
  rng = np.random.RandomState(seed)
  r = np.array(radius_zyx)
  paths = []
  for ida, idb, (x, y, z) in points:
    c = np.array([z, y, x])
    if np.any(c - r < 0) or np.any(c + r + 1 > np.array(seg.shape)):
      continue
    box = seg[c[0] - r[0]:c[0] + r[0] + 1, c[1] - r[1]:c[1] + r[1] + 1, c[2] - r[2]:c[2] + r[2] + 1]
    probs, dels, hist, starts = [], [], [], np.empty(2, dtype=object)
    merge = rng.rand() < 0.5
    for k, sid in enumerate((ida, idb)):
      mask = _grow(box == sid, rng.randint(0, 3))
      if merge:
        mask |= box == (idb if k == 0 else ida)
      q = np.where(mask, rng.randint(128, 256, box.shape), rng.randint(1, 128, box.shape)).astype(np.uint8)
      q[rng.rand(*box.shape) < 0.02] = 0
      probs.append(q)
      steps = rng.randint(3, 13)
      dels.append(rng.randint(0, 500, steps).astype(np.int64))
      hist.append(rng.randint(0, 2 * r + 1, (steps, 3)).astype(np.int32))
      starts[k] = rng.randint(0, 2 * r + 1, (rng.randint(1, 4), 3))
    ragged = lambda items: np.array(items) if len({len(i) for i in items}) == 1 else _objects(items)  # noqa: E731
    path = os.path.join(directory, '%d-%d_at_%d_%d_%d.npz' % (ida, idb, x, y, z))
    np.savez_compressed(path, probs=np.stack(probs), deletes=ragged(dels), histories=ragged(hist), start_points=starts)
    paths.append(path)
  return paths


def _objects(items):
  out = np.empty(len(items), dtype=object)
  for k, it in enumerate(items):
    out[k] = it
  return out
