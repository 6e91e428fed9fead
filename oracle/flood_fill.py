"""Oracle: flood-fill inference loop on the CPU (test infrastructure; see oracle/__init__.py).

A compact numpy restatement of the reference's per-object and per-canvas loops:

* ffn/inference/inference.py:186-195  thresholds -> logits, stored back as float32
* ffn/inference/inference.py:312-346  Canvas.is_valid_pos
* ffn/inference/inference.py:386-441  Canvas.update_at (NaN->pad, predict, disco merge, paste)
* ffn/inference/inference.py:443-450  Canvas.init_seed
* ffn/inference/inference.py:460-533  Canvas.segment_at
* ffn/inference/inference.py:538-683  Canvas.segment_all
* ffn/inference/movement.py:42-100    get_scored_move_offsets
* ffn/inference/movement.py:166-222   FaceMaxMovementPolicy (BFS deque + quantised done-set)
* ffn/inference/movement.py:225-244   get_policy_fn (float64 policy threshold)
* ffn/inference/storage.py:137-143    quantize_probability

All coordinates are (z, y, x).  The network is injected as ``net(seed_patch, image_patch) ->
logits`` so the same loop can be driven by the CPU conv stack (pure oracle) or by the CUDA
engine's ``predict`` (to check the device-side loop logic bit-exactly).
"""

from __future__ import annotations

import collections
import dataclasses
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
from scipy.special import expit, logit


@dataclasses.dataclass
class Options:
  """InferenceOptions in probability space (ffn/inference/inference.proto:131-168)."""
  init_activation: float = 0.95
  pad_value: float = 0.05
  move_threshold: float = 0.9
  segment_threshold: float = 0.6
  disco_seed_threshold: float = 0.0     # proto2 default of an unset float field
  min_boundary_dist: Tuple[int, int, int] = (1, 1, 1)   # z, y, x
  min_segment_size: int = 1000
  # FaceMaxMovementPolicy's score_threshold (logit space, float64), as set by
  # InferenceRequest.movement_policy_args; None is get_policy_fn's logit(move_threshold)
  policy_score_threshold: Optional[float] = None


def f32_logit(p: float) -> np.float32:
  """What ends up in the float32 proto field after inference.py:186-195."""
  return np.float32(logit(float(np.float32(p))))


def policy_threshold(move_threshold_prob: float) -> float:
  """movement.py:241-242: float64 logit of the float32 proto value."""
  return float(logit(float(np.float32(move_threshold_prob))))


def quantize_probability(prob: np.ndarray) -> np.ndarray:
  """storage.py:137-143."""
  q = np.digitize(prob, np.linspace(0.0, 1.0, 255))
  q[np.isnan(prob)] = 0
  return q.astype(np.uint8)


def scored_moves(deltas, logits: np.ndarray, threshold: float):
  """movement.py:42-100 — best voxel on each of the (up to) six faces at +-delta.

  Returns a list of (score: np.float32, (dz, dy, dx)) with score compared against `threshold`
  in float64 (NumPy<2 semantics; identical to the float32 compare for every threshold whose
  nearest float32 is >= it, which holds for the reference's 0.9 / 0.6 — SURVEY.md 8a row 6).
  """
  c = [s // 2 for s in logits.shape]
  lo = [ci - d for ci, d in zip(c, deltas)]
  hi = [ci + d + 1 for ci, d in zip(c, deltas)]
  out = []
  for axis in range(3):
    d = int(deltas[axis])
    if d == 0:
      continue
    for off in (-d, d):
      sl = [slice(lo[a], hi[a]) for a in range(3)]
      sl[axis] = c[axis] + off
      face = logits[tuple(sl)]
      flat = int(face.argmax())                  # first maximum in C order
      fpos = np.unravel_index(flat, face.shape)
      score = face[fpos]
      if float(score) < threshold:
        continue
      rel = [int(fpos[0]) - face.shape[0] // 2, int(fpos[1]) - face.shape[1] // 2]
      rel.insert(axis, off)
      item = (score, tuple(rel))
      if item not in out:
        out.append(item)
  return out


class FaceMaxPolicy:
  """movement.py:166-222."""

  def __init__(self, canvas: 'Canvas', deltas, score_threshold: float):
    self.canvas = canvas
    self.deltas = np.asarray(deltas, dtype=np.int64)
    self.score_threshold = score_threshold
    self.reset(None)

  def reset(self, start_pos):
    self.queue = collections.deque()
    self.done = set()
    self.start = None if start_pos is None else np.asarray(start_pos, dtype=np.int64)

  def quantize(self, pos):
    rel = np.asarray(pos, dtype=np.int64) - self.start
    return tuple(int(v) for v in (rel + self.deltas // 2) // np.maximum(self.deltas, 1))

  def pop(self):
    """movement.py:186-198; returns None when the queue is exhausted."""
    while self.queue:
      _, coord = self.queue.popleft()
      coord = tuple(int(v) for v in coord)
      if self.quantize(coord) in self.done:
        continue
      if self.canvas.is_valid_pos(coord):
        return coord
    return None

  def update(self, logits, pos):
    """movement.py:210-222."""
    self.done.add(self.quantize(pos))
    moves = scored_moves(self.deltas, logits, self.score_threshold)
    moves.sort(reverse=True)                     # descending by (score, (dz,dy,dx))
    for score, rel in moves:
      self.queue.append((score, tuple(int(p) + int(r) for p, r in zip(pos, rel))))


class Canvas:
  """Restated ffn.inference.inference.Canvas (state + loops only; no I/O, no executor)."""

  def __init__(self, net: Callable[[np.ndarray, np.ndarray], np.ndarray], image: np.ndarray,
               fov_zyx: Sequence[int], deltas_zyx: Sequence[int], options: Options,
               keep_probability_maps: bool = True, mask: Optional[np.ndarray] = None,
               seed_mask: Optional[np.ndarray] = None):
    self.net = net
    self.image = np.asarray(image, dtype=np.float32)
    self.shape = self.image.shape
    self.fov = np.asarray(fov_zyx, dtype=np.int64)
    self.margin = self.fov // 2
    self.opt = options
    # inference.py:186-195
    self.init_activation = f32_logit(options.init_activation)
    self.pad_value = f32_logit(options.pad_value)
    self.move_threshold = f32_logit(options.move_threshold)
    self.segment_threshold = f32_logit(options.segment_threshold)
    self.disco_seed_threshold = float(np.float32(options.disco_seed_threshold))

    self.seed = np.full(self.shape, np.nan, dtype=np.float32)
    self.segmentation = np.zeros(self.shape, dtype=np.int32)
    self.seg_prob = np.zeros(self.shape, dtype=np.uint8) if keep_probability_maps else None
    self.mask = mask            # MovementRestrictor.mask (movement.py:303-314)
    self.seed_mask = seed_mask  # MovementRestrictor.seed_mask (movement.py:290-301)
    score_threshold = options.policy_score_threshold
    if score_threshold is None:
      score_threshold = policy_threshold(options.move_threshold)
    self.policy = FaceMaxPolicy(self, deltas_zyx, float(score_threshold))
    self.max_id = 0
    self.origins: Dict[int, Tuple[Tuple[int, int, int], int]] = {}
    self.overlaps: Dict[int, np.ndarray] = {}
    self.counters = collections.Counter()
    self.min_pos = np.zeros(3, np.int64)
    self.max_pos = np.zeros(3, np.int64)
    # Diagnostics for the parity report.
    self.trace: List[Tuple[int, int, int]] = []      # every FoV position, in order
    self.history: List[Tuple[int, int, int]] = []    # Canvas.history of the current object
    self.history_deleted: List[int] = []             # Canvas.history_deleted of the current object
    self.disco_applied: List[bool] = []              # per FoV step (all objects): was the disco merge applied
    self.min_margin = float('inf')                   # closest |value - threshold| of any decision

  # -- helpers ------------------------------------------------------------------------------

  def _fov_sel(self, pos):
    lo = np.asarray(pos, dtype=np.int64) - self.margin
    return tuple(slice(int(a), int(a + s)) for a, s in zip(lo, self.fov))

  def _note_margin(self, value, threshold):
    if np.isfinite(value):
      self.min_margin = min(self.min_margin, abs(float(value) - float(threshold)))

  def is_valid_pos(self, pos, ignore_move_threshold=False) -> bool:
    """inference.py:312-346."""
    pos = tuple(int(p) for p in pos)
    if not ignore_move_threshold:
      v = self.seed[pos]
      self._note_margin(v, self.move_threshold)
      if v < self.move_threshold:
        self.counters['skip_threshold'] += 1
        return False
    p = np.asarray(pos, dtype=np.int64)
    if np.any(p - self.margin < 0) or np.any(p + self.margin >= np.asarray(self.shape)):
      self.counters['skip_invalid_pos'] += 1
      return False
    if self.segmentation[pos] > 0:
      self.counters['skip_invalid_pos'] += 1
      return False
    return True

  # -- single step --------------------------------------------------------------------------

  def update_at(self, pos) -> np.ndarray:
    """inference.py:386-441 with pred size == seed size (_pred_delta = 0)."""
    sel = self._fov_sel(pos)
    old = self.seed[sel]
    fed = old.copy()
    fed[np.isnan(fed)] = self.pad_value
    logits = np.array(self.net(fed, self.image[sel]), dtype=np.float32)
    self.counters['inference-calls'] += 1

    merge = False
    if self.disco_seed_threshold >= 0:
      # Canvas.history_deleted (inference.py:420-422; kept unconditionally here, the reference keeps it
      # under keep_history): float32 old seed against the float64 logit(0.8), raw logits against logit(0.5)
      with np.errstate(invalid='ignore'):
        self.history_deleted.append(int(np.sum((old >= 1.3862943611198908) & (logits < 0.0))))
      merge = bool(np.mean(logits >= self.move_threshold) > self.disco_seed_threshold)
      if merge:
        with np.errstate(invalid='ignore'):
          keep_old = (old < np.float32(0.0)) & (logits > old)   # logit(0.5) == 0
        logits[keep_old] = old[keep_old]
    self.disco_applied.append(merge)
    self.seed[sel] = logits
    return logits

  def init_seed(self, pos):
    """inference.py:443-450."""
    self.seed[...] = np.nan
    self.seed[tuple(pos)] = self.init_activation

  # -- one object ---------------------------------------------------------------------------

  def segment_at(self, start_pos) -> int:
    """inference.py:460-533 (partial_segment_iters == 0, reset_seed_per_segment == True)."""
    start_pos = tuple(int(p) for p in start_pos)
    self.init_seed(start_pos)
    self.policy.reset(start_pos)
    self.history, self.history_deleted = [], []     # reset_state (inference.py:303-304)
    self.min_pos = np.asarray(start_pos, dtype=np.int64)
    self.max_pos = np.asarray(start_pos, dtype=np.int64)
    self.policy.queue.append((self.policy.score_threshold * 2, start_pos))

    iters = 0
    while True:
      pos = self.policy.pop()
      if pos is None:
        break
      v0 = self.seed[start_pos]
      self._note_margin(v0, self.move_threshold)
      if v0 < self.move_threshold:
        self.counters['seed_got_too_weak'] += 1
        break
      if self.mask is not None and self.mask[pos]:
        self.counters['skip_restriced_pos'] += 1
        continue
      logits = self.update_at(pos)
      self.trace.append(pos)
      self.history.append(pos)                        # inference.py:520-521
      self.min_pos = np.minimum(self.min_pos, pos)
      self.max_pos = np.maximum(self.max_pos, pos)
      iters += 1
      for axis_moves in scored_moves(self.policy.deltas, logits, -np.inf):
        self._note_margin(axis_moves[0], self.policy.score_threshold)
      self.policy.update(logits, pos)
    return iters

  # -- whole canvas -------------------------------------------------------------------------

  def segment_all(self, seeds: Sequence[Sequence[int]]):
    """inference.py:538-683 with the seed policy replaced by an explicit (z,y,x) list.

    The list plays the role of `BaseSeedPolicy.coords` *after* the border filter of
    seed.py:81-88, which is re-applied here for safety (it is idempotent).
    """
    mbd = np.asarray(self.opt.min_boundary_dist, dtype=np.int64)
    shape = np.asarray(self.shape)
    for pos in seeds:
      pos = tuple(int(p) for p in pos)
      p = np.asarray(pos, dtype=np.int64)
      if np.any(p - self.margin < 0) or np.any(p + self.margin >= shape):
        continue                                        # seed.py:81-88 (never reaches the canvas)
      self.counters['seeds-examined'] += 1
      if not self.is_valid_pos(pos, ignore_move_threshold=True):
        continue
      if self.mask is not None and self.mask[pos]:
        continue
      if self.seed_mask is not None and self.seed_mask[pos]:
        continue
      lo, hi = p - mbd, p + mbd + 1
      if np.any(self.segmentation[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] > 0):
        self.segmentation[pos] = -1
        continue

      iters = self.segment_at(pos)
      self.counters['segment_at-calls'] += 1
      if iters <= 0:
        continue
      if self.seed[pos] < self.move_threshold:
        if self.segmentation[pos] == 0:
          self.segmentation[pos] = -1
        self.counters['invalid-weak'] += 1
        continue

      half = self.fov // 2
      lo = np.maximum(self.min_pos - half, 0)
      hi = self.max_pos + half + 1
      sel = tuple(slice(int(a), int(b)) for a, b in zip(lo, hi))
      mask = self.seed[sel] >= self.segment_threshold
      raw = int(mask.sum())
      ids, counts = np.unique(self.segmentation[sel][mask], return_counts=True)
      keep = ids > 0
      ids, counts = ids[keep], counts[keep]
      mask &= self.segmentation[sel] <= 0
      actual = int(mask.sum())
      if actual < self.opt.min_segment_size:
        if self.segmentation[pos] == 0:
          self.segmentation[pos] = -1
        self.counters['invalid-small'] += 1
        continue

      self.counters['voxels-segmented'] += actual
      self.counters['voxels-overlapping'] += raw - actual
      self.max_id += 1
      while self.max_id in self.origins:
        self.max_id += 1
      sid = self.max_id
      self.segmentation[sel][mask] = sid
      if self.seg_prob is not None:
        self.seg_prob[sel][mask] = quantize_probability(expit(self.seed[sel][mask]))
      self.overlaps[sid] = np.array([ids, counts])
      self.origins[sid] = (pos, iters)


def grid_seeds(shape_zyx, step=16, offsets=(0, 8, 4, 12, 2, 10, 14)):
  """seed.py:411-430 PolicyGrid3d.init_coords (exactly restatable: pure index arithmetic)."""
  out = []
  for off in offsets:
    for z in range(off, shape_zyx[0], step):
      for y in range(off, shape_zyx[1], step):
        for x in range(off, shape_zyx[2], step):
          out.append((z, y, x))
  return np.asarray(out, dtype=np.int64).reshape(-1, 3)


def canonical_relabel(seg: np.ndarray) -> np.ndarray:
  """Maps labels > 0 to their rank of first occurrence in C-order raster scan (SURVEY.md 8c)."""
  flat = np.asarray(seg).ravel()
  ids, first = np.unique(flat, return_index=True)
  keep = ids > 0
  ids, first = ids[keep], first[keep]
  rank = np.empty(len(ids), dtype=np.int64)
  rank[np.argsort(first, kind='stable')] = np.arange(1, len(ids) + 1)
  out = np.zeros(flat.shape, dtype=np.int64)
  positive = flat > 0
  out[positive] = rank[np.searchsorted(ids, flat[positive])]
  return out.reshape(np.asarray(seg).shape)
