"""Scoring of resegmentation results on the device: ffn/inference/resegmentation_analysis.py.

`process_point` (resegmentation.py) leaves one result file per decision point.  The functions here turn such a
file and the original segmentation into the reference's `PairResegmentationResult` / `EndpointResegmentationResult`
protos, with the reference's names and signatures.  The batched forms score many files with one device call:
file reading and the segmentation crops run on a thread pool, the per-voxel work (masks, counts, exact Euclidean
distance transforms, overlap counts) in libffn_b200 (`ffn_reseg_eval`).  There is no host fallback.

`seg_volume` is indexed as the reference indexes it, `seg_volume[0, z0:z1, y0:y1, x0:x1][0, ...]`, where a volume
store keeps the channel axis; a numpy array, which drops it, works too.  Voxel sizes must be positive integers: the
distances are then exact integers on the device, and `float(np.sqrt(D))` is what scipy's `distance_transform_edt` returns for them.  A mask without any voxel outside it
in the box gets what scipy returns there (see `ffn_reseg_eval` in include/ffn_b200.h).
"""

from __future__ import annotations

import ctypes as C
import logging
import re

import numpy as np

from ffn_b200 import _lib
from . import resegmentation_pb2
from . import storage


class InvalidBaseSegmentatonError(Exception):
  pass


class IncompleteResegmentationError(Exception):
  pass


# Mask voxels per device call (four masks per pair item): bounds the device memory of one call to about 1.6 GB.
_MAX_MASK_VOXELS = 1 << 26


def compute_iou(reseg):
  """Jaccard index of the two objects of a [2, z, y, x] boolean array."""
  return (np.sum(reseg[0, ...] & reseg[1, ...]) /
          float(np.sum(np.max(reseg, axis=0))))


def parse_resegmentation_filename(filename):
  logging.info('processing: %s', filename)
  id1, id2, x, y, z = [
      int(t) for t in
      re.search(r'(\d+)-(\d+)_at_(\d+)_(\d+)_(\d+)', filename).groups()]
  return id1, id2, x, y, z


def _voxel_size(voxel_size):
  vs = tuple(voxel_size)
  if len(vs) != 3:
    raise ValueError('voxel_size must have 3 components (z, y, x), got %r' % (voxel_size,))
  out = []
  for v in vs:
    try:
      ok = int(v) == v and 0 < int(v) < 2**31
    except (TypeError, ValueError, OverflowError):
      ok = False
    if not ok:
      raise ValueError('voxel sizes must be positive integers below 2^31, got %r' % (voxel_size,))
    out.append(int(v))
  return tuple(out)


def _mask_table(threshold):
  """q -> (nan_to_num(dequantize_probability(q)) >= threshold), by the same numpy operations as on a whole box."""
  prob = np.nan_to_num(storage.dequantize_probability(np.arange(256, dtype=np.uint8)))
  return np.ascontiguousarray(prob >= threshold, dtype=np.uint8)


def _read(filename, keys):
  with open(filename, 'rb') as f:
    data = np.load(f, allow_pickle=True)   # ragged start points / histories are object arrays
    return [data[k] for k in keys]


def _crop(seg_volume, center_zyx, radius_zyx):
  """seg_volume[0, box] as the reference reads it; [1, z, y, x] (a volume store) or [z, y, x] (a numpy array)."""
  z, y, x = center_zyx
  rz, ry, rx = radius_zyx
  crop = np.asarray(seg_volume[0, (z - rz):(z + rz + 1), (y - ry):(y + ry + 1), (x - rx):(x + rx + 1)])
  return crop[0, ...] if crop.ndim == 4 else crop


def _box_array(a, shape, what, filename):
  a = np.asarray(a)
  if a.shape != tuple(shape):
    raise ValueError('%s of %s has shape %r, expected %r' % (what, filename, a.shape, tuple(shape)))
  return a


def _run(pair, box, voxel_size, table, items, device):
  """Device call(s) over `items` = [(labels, probs [k, box], id_a, id_b)]: FfnResegStats and, for endpoints, the
  overlap rows of each item."""
  nbox = int(np.prod(box))
  per_call = max(1, _MAX_MASK_VOXELS // (nbox * (4 if pair else 1)))
  stats = np.zeros(len(items), dtype=_lib.RESEG_STATS_DTYPE)
  rows = [None] * len(items)
  if not items:
    return stats, rows
  lib = _lib.load()
  for lo in range(0, len(items), per_call):
    chunk = items[lo:lo + per_call]
    labels = np.stack([it[0] for it in chunk]).astype(np.uint64, copy=False)
    probs = np.stack([it[1] for it in chunk]).astype(np.uint8, copy=False)
    ids = np.array([[it[2], it[3]] for it in chunk], dtype=np.uint64)
    labels, probs = np.ascontiguousarray(labels), np.ascontiguousarray(probs)
    desc = _lib.ResegEvalDesc()
    desc.box_zyx[:] = box
    desc.voxel_size_zyx[:] = voxel_size
    desc.pair = int(pair)
    desc.num_items = len(chunk)
    out = stats[lo:lo + len(chunk)]   # a view: filled in place
    cap = 0 if pair else 64 * len(chunk)
    while True:
      ov = np.zeros(max(cap, 1), dtype=_lib.RESEG_OVERLAP_DTYPE)
      n = C.c_int64(0)
      _lib.check(lib.ffn_reseg_eval(int(device), C.byref(desc), _lib.ptr(labels), _lib.ptr(probs), _lib.ptr(ids),
                                    _lib.ptr(table), _lib.ptr(out), _lib.ptr(ov), cap, C.byref(n)))
      if n.value <= cap:
        break
      cap = n.value
    if not pair:
      ov = ov[:n.value]
      bounds = np.searchsorted(ov['item'], np.arange(len(chunk) + 1))
      for k in range(len(chunk)):
        rows[lo + k] = ov[bounds[k]:bounds[k + 1]]
  return stats, rows


def _load_pair(filename, seg_volume, resegmentation_radius, analysis_radius):
  """Host part of evaluate_pair_resegmentation up to the per-voxel work: (result, labels, probs, dels, moves, delta)."""
  id1, id2, x, y, z = parse_resegmentation_filename(filename)
  result = resegmentation_pb2.PairResegmentationResult()
  result.id_a, result.id_b = id1, id2
  p = result.point
  p.x, p.y, p.z = x, y, z
  sr = result.segmentation_radius
  sr.z, sr.y, sr.x = resegmentation_radius

  prob, dels, moves, start_points = _read(filename, ('probs', 'deletes', 'histories', 'start_points'))
  if prob.shape[0] != 2:
    raise IncompleteResegmentationError()
  assert prob.ndim == 4

  # The last start point of each object counts (x, y, z, relative to the resegmentation box).
  corner = np.array([p.x - sr.x, p.y - sr.y, p.z - sr.z])
  for src, origin in ((start_points[0], result.eval.from_a.origin), (start_points[1], result.eval.from_b.origin)):
    origin.x, origin.y, origin.z = np.array(src[-1], dtype=int) + corner

  analysis_r = np.array(analysis_radius)
  r = result.eval.radius
  r.z, r.y, r.x = analysis_r
  box = tuple(int(v) for v in 2 * analysis_r + 1)
  seg = _box_array(_crop(seg_volume, (z, y, x), analysis_r), box, 'segmentation crop', filename)
  delta = np.array(resegmentation_radius) - analysis_r
  prob = _box_array(prob[:, delta[0]:(delta[0] + 2 * analysis_r[0] + 1),
                         delta[1]:(delta[1] + 2 * analysis_r[1] + 1),
                         delta[2]:(delta[2] + 2 * analysis_r[2] + 1)], (2,) + box, 'analysis box of probs', filename)
  return result, seg, prob, dels, moves, delta


def _deleted_voxels(dels, moves, delta, analysis_r):
  """Sum of `dels` over the FoV moves that lie inside the analysis box (None: no moves recorded)."""
  if moves.size == 0:
    return None
  corner0_zyx = np.array(delta)
  corner1_zyx = np.array(delta) + 2 * np.array(analysis_r)
  mask = np.all((moves >= corner0_zyx[np.newaxis, ...]) & (moves <= corner1_zyx[np.newaxis, ...]), axis=1)
  return int(np.sum(dels[mask]))


def _fill_segment_result(result, k, s, dels, moves, delta, analysis_r):
  result.max_edt = float(np.sqrt(np.float64(s['max_edt2'][2 + k])))
  deleted = _deleted_voxels(dels, moves, delta, analysis_r)
  if deleted is not None:
    result.deleted_voxels = deleted
  result.num_voxels = int(s['n_reseg'][k])
  result.segment_a_consistency = float(s['n_reseg_seg'][k][0]) / np.int64(s['n_seg'][0])
  result.segment_b_consistency = float(s['n_reseg_seg'][k][1]) / np.int64(s['n_seg'][1])


def _gather(fn, filenames):
  """fn(filename) for every file on the I/O thread pool, in input order; the two analysis errors become values."""
  def run(filename):
    try:
      return fn(filename)
    except (InvalidBaseSegmentatonError, IncompleteResegmentationError) as e:
      return e
  return list(storage._pool().map(run, filenames))   # pylint: disable=protected-access


def evaluate_pair_resegmentations(filenames, seg_volume, resegmentation_radius, analysis_radius, voxel_size,
                                  threshold=0.5, device=0):
  """evaluate_pair_resegmentation of every file, with one device call per batch.

  Returns a list in input order: a PairResegmentationResult per file, or the InvalidBaseSegmentatonError /
  IncompleteResegmentationError instance that file raised.  Input the reference cannot score at all raises for the
  whole batch: a ValueError when a segmentation crop or analysis box of probabilities does not have the analysis box's
  extent (a point whose box crosses the volume edge; the reference fails there with an IndexError), even if that
  file's ids are missing too.
  """
  vs = _voxel_size(voxel_size)
  analysis_r = np.array(analysis_radius)
  box = tuple(int(v) for v in 2 * analysis_r + 1)
  loaded = _gather(lambda f: _load_pair(f, seg_volume, resegmentation_radius, analysis_radius), list(filenames))
  todo = [k for k, it in enumerate(loaded) if not isinstance(it, Exception)]
  stats, _ = _run(True, box, vs, _mask_table(threshold),
                  [(loaded[k][1], loaded[k][2], loaded[k][0].id_a, loaded[k][0].id_b) for k in todo], device)
  out = list(loaded)
  for k, s in zip(todo, stats):
    result, _, _, dels, moves, delta = loaded[k]
    e = result.eval
    e.num_voxels_a = int(s['n_seg'][0])
    e.num_voxels_b = int(s['n_seg'][1])
    if e.num_voxels_a == 0 or e.num_voxels_b == 0:
      out[k] = InvalidBaseSegmentatonError()
      continue
    e.max_edt_a = float(np.sqrt(np.float64(s['max_edt2'][0])))
    e.max_edt_b = float(np.sqrt(np.float64(s['max_edt2'][1])))
    with np.errstate(invalid='ignore', divide='ignore'):   # two empty objects: nan, as compute_iou
      e.iou = np.int64(s['n_inter']) / float(s['n_union'])
    _fill_segment_result(e.from_a, 0, s, dels[0], moves[0], delta, analysis_r)
    _fill_segment_result(e.from_b, 1, s, dels[1], moves[1], delta, analysis_r)
    out[k] = result
  return out


def _load_endpoint(filename, seg_volume, resegmentation_radius):
  id1, _, x, y, z = parse_resegmentation_filename(filename)
  result = resegmentation_pb2.EndpointSegmentationResult()
  result.id = id1
  start = result.start
  start.x, start.y, start.z = x, y, z
  sr = result.segmentation_radius
  sr.z, sr.y, sr.x = resegmentation_radius
  prob, = _read(filename, ('probs',))
  orig_seg = _crop(seg_volume, (z, y, x), (sr.z, sr.y, sr.x))
  if np.issubdtype(orig_seg.dtype, np.signedinteger) and orig_seg.size and orig_seg.min() < 0:
    raise ValueError('%s: the segmentation box holds negative ids, which overlap maps (uint64 keys) cannot hold'
                     % filename)
  return result, orig_seg, _box_array(prob[:1], (1,) + orig_seg.shape, 'probs', filename)


def evaluate_endpoint_resegmentations(filenames, seg_volume, resegmentation_radius, threshold=0.5, device=0):
  """evaluate_endpoint_resegmentation of every file, with one device call per batch of equal box extents.

  Returns a list in input order: an EndpointResegmentationResult per file, or the InvalidBaseSegmentatonError
  instance that file raised.  Input the reference cannot score at all raises for the whole batch: a ValueError when a
  segmentation crop does not have the extent of the file's probability map (a point whose box crosses the volume
  edge), or when it holds negative ids, which the uint64 keys of the overlap map cannot hold.
  """
  loaded = _gather(lambda f: _load_endpoint(f, seg_volume, resegmentation_radius), list(filenames))
  out = list(loaded)
  by_box = {}
  for k, it in enumerate(loaded):
    if not isinstance(it, Exception):
      by_box.setdefault(it[1].shape, []).append(k)
  table = _mask_table(threshold)
  for box, todo in by_box.items():
    stats, rows = _run(False, box, (0, 0, 0), table,
                       [(loaded[k][1], loaded[k][2], loaded[k][0].id, 0) for k in todo], device)
    for k, s, r in zip(todo, stats, rows):
      result = loaded[k][0]
      if s['n_seg'][0] == 0:
        out[k] = InvalidBaseSegmentatonError()
        continue
      result.num_voxels = int(s['n_reseg'][0])
      for old, v, n in zip(r['id'], r['num_overlapping'], r['num_original']):
        old = int(old)
        result.overlaps[old].num_overlapping = int(v)
        result.overlaps[old].num_original = int(n)
        if old == result.id:
          result.source.CopyFrom(result.overlaps[old])
      out[k] = result
  return out


def _single(results):
  if isinstance(results[0], Exception):
    raise results[0]
  return results[0]


def evaluate_pair_resegmentation(filename, seg_volume, resegmentation_radius, analysis_radius, voxel_size,
                                 threshold=0.5, device=0):
  """Evaluates segment pair resegmentation (resegmentation_analysis.py:159-260).

  Args:
    filename: path to the file containing resegmentation results
    seg_volume: 4-d array-like with the original segmentation
    resegmentation_radius: (z, y, x) radius of the resegmentation subvolume
    analysis_radius: (z, y, x) radius of the subvolume in which to perform analysis
    voxel_size: (z, y, x) voxel size in physical units; positive integers
    threshold: threshold at which to create objects from the predicted object map
    device: CUDA device index (an H100)

  Returns:
    PairResegmentationResult proto

  Raises:
    IncompleteResegmentationError: when the resegmentation data does not represent two finished segments
    InvalidBaseSegmentatonError: when no base segmentation object with the expected ID matches the data
  """
  return _single(evaluate_pair_resegmentations([filename], seg_volume, resegmentation_radius, analysis_radius,
                                               voxel_size, threshold, device))


def evaluate_endpoint_resegmentation(filename, seg_volume, resegmentation_radius, threshold=0.5, device=0):
  """Evaluates endpoint resegmentation (resegmentation_analysis.py:97-156).

  Args:
    filename: path to the file containing resegmentation results
    seg_volume: 4-d array-like with the original segmentation
    resegmentation_radius: (z, y, x) radius of the resegmentation subvolume
    threshold: threshold at which to create objects from the predicted object map
    device: CUDA device index (an H100)

  Returns:
    EndpointResegmentationResult proto

  Raises:
    InvalidBaseSegmentatonError: when no base segmentation object with the expected ID matches the data
  """
  return _single(evaluate_endpoint_resegmentations([filename], seg_volume, resegmentation_radius, threshold, device))


def evaluate_segmentation_result(reseg, dels, moves, delta, analysis_r, seg1, seg2, sampling, result, device=0):
  """Fills a SegmentResult from one resegmented object (resegmentation_analysis.py:52-86), on the device.

  reseg, seg1, seg2: 3d boolean masks of one box (seg1 and seg2 disjoint); dels, moves: per FoV step deleted voxels
  and (z, y, x) positions; delta, analysis_r: offset and radius of the analysis box; sampling: integer voxel size;
  device: CUDA device index (an H100).
  """
  reseg, seg1, seg2 = (np.asarray(a, dtype=bool) for a in (reseg, seg1, seg2))
  if np.any(seg1 & seg2):
    raise ValueError('seg1 and seg2 must be disjoint')
  labels = seg1.astype(np.uint64) + 2 * seg2.astype(np.uint64)
  probs = np.stack([reseg, np.zeros_like(reseg)]).astype(np.uint8)
  table = np.zeros(256, dtype=np.uint8)
  table[1] = 1
  stats, _ = _run(True, reseg.shape, _voxel_size(sampling), table, [(labels, probs, 1, 2)], device)
  _fill_segment_result(result, 0, stats[0], np.asarray(dels), np.asarray(moves), delta, analysis_r)
