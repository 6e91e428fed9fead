"""FoV movement: host-side mirror of the policy objects whose state lives on the device.

The per-step evaluation (face arg-max, threshold, descending sort, queue push/pop, quantised
done-set) runs inside the persistent kernel (ffn_b200/csrc/flood_kernel.cuh: policy_finish,
warp_pop).  This module keeps the reference's public surface — ffn/inference/movement.py:
`get_scored_move_offsets` (:42-100), `BaseMovementPolicy` (:103-163), `FaceMaxMovementPolicy`
(:166-222), `get_policy_fn` (:225-244), `MovementRestrictor` (:247-336) — so callers,
checkpoints and request protos keep working.  `get_scored_move_offsets` is provided as a host
utility for callers that inspect prediction patches themselves; the engine never calls it.
"""

import collections
import json
import weakref

import numpy as np
from scipy.special import logit


def get_scored_move_offsets(deltas, prob_map, threshold=0.9):
  """Yields (score, (dz, dy, dx)) for the best voxel on each face at +-deltas."""
  center = np.array(prob_map.shape) // 2
  assert center.size == 3
  box = [slice(int(c - d), int(c + d + 1)) for c, d in zip(center, deltas)]
  seen = set()
  for axis, delta in enumerate(deltas):
    if delta == 0:
      continue
    for off in (-delta, delta):
      sel = list(box)
      sel[axis] = int(center[axis] + off)
      face = prob_map[tuple(sel)]
      pos = np.unravel_index(face.argmax(), face.shape)
      score = face[pos]
      if score < threshold:
        continue
      rel = [int(pos[0]) - face.shape[0] // 2, int(pos[1]) - face.shape[1] // 2]
      rel.insert(axis, int(off))
      item = (score, tuple(rel))
      if item not in seen:
        seen.add(item)
        yield item


class BaseMovementPolicy:
  """Base class of movement policies (interface only; see FaceMaxMovementPolicy)."""

  def __init__(self, canvas, scored_coords, deltas):
    self.canvas = weakref.proxy(canvas)
    self.scored_coords = scored_coords
    self.deltas = np.array(deltas)

  def __len__(self):
    return len(self.scored_coords)

  def __iter__(self):
    return self

  def __next__(self):
    raise StopIteration()

  def next(self):
    return self.__next__()

  def append(self, item):
    self.scored_coords.append(item)

  def update(self, prob_map, position):
    raise NotImplementedError()

  def get_state(self):
    raise NotImplementedError()

  def restore_state(self, state):
    raise NotImplementedError()

  def reset_state(self, start_pos):
    raise NotImplementedError()


class FaceMaxMovementPolicy(BaseMovementPolicy):
  """Face-maximum BFS policy.  The live deque / done-set are device-resident; `scored_coords`,
  `done_rounded_coords` and `get_state` pull a snapshot, `restore_state` pushes one."""

  def __init__(self, canvas, deltas=(4, 8, 8), score_threshold=0.9):
    self.score_threshold = score_threshold
    self._start_pos = None
    super().__init__(canvas, collections.deque([]), deltas)
    self.done_rounded_coords = set()

  def _device(self):
    return getattr(self.canvas, '_dev', None)

  def reset_state(self, start_pos):
    self.scored_coords = collections.deque([])
    self.done_rounded_coords = set()
    self._start_pos = start_pos

  def sync_from_device(self):
    dev = self._device()
    if dev is None:
      return
    queue, done, start = dev.policy_state()
    self.scored_coords = collections.deque(
        (np.float32(q[0]), (int(q[1]), int(q[2]), int(q[3]))) for q in queue)
    self.done_rounded_coords = set(tuple(int(v) for v in d) for d in done)
    self._start_pos = start

  def get_state(self):
    self.sync_from_device()
    return [(self.scored_coords, self.done_rounded_coords, self._start_pos)]

  def restore_state(self, state):
    self.scored_coords, self.done_rounded_coords, self._start_pos = state[0]
    dev = self._device()
    if dev is not None and self._start_pos is not None:
      queue = np.asarray([(float(s),) + tuple(int(v) for v in c) for s, c in self.scored_coords],
                         dtype=np.float64).reshape(-1, 4)
      done = np.asarray(sorted(self.done_rounded_coords), dtype=np.int32).reshape(-1, 3)
      dev.set_policy_state(queue, done, self._start_pos)

  def quantize_pos(self, pos):
    rel_pos = np.array(pos) - self._start_pos
    return tuple((rel_pos + self.deltas // 2) // np.maximum(self.deltas, 1))


def get_policy_fn(request, model_info):
  """Policy factory from an InferenceRequest (movement.py:225-244).

  Only FaceMaxMovementPolicy (the default) runs on the device; other names are rejected when
  the canvas is built.
  """
  name = request.movement_policy_name or 'FaceMaxMovementPolicy'
  if name.split('.')[-1] != 'FaceMaxMovementPolicy':
    raise NotImplementedError('movement policy %r has no device implementation' % name)
  kwargs = json.loads(request.movement_policy_args) if request.movement_policy_args else {}
  if 'deltas' not in kwargs:
    kwargs['deltas'] = model_info.deltas[::-1]
  if 'score_threshold' not in kwargs:
    kwargs['score_threshold'] = logit(request.inference_options.move_threshold)
  return lambda canvas: FaceMaxMovementPolicy(canvas, **kwargs)


class MovementRestrictor:
  """Excludes areas from segmentation (movement.py:247-336).

  `mask` and `seed_mask` live on the device next to the canvas.  A shift mask (a 2-d shift vector field per
  section: positions whose FoV box contains a shift component >= `shift_mask_threshold` are not entered,
  :312-334) is folded on the host into the per-voxel movement mask the device loop consults
  (`movement_mask`): `is_valid_pos` is a pure function of the position, so evaluating it for every voxel
  once gives the device exactly the reference's verdicts (and the same 'skip_restriced_pos' counts).
  """

  def __init__(self, mask=None, shift_mask=None, shift_mask_fov=None, shift_mask_threshold=4,
               shift_mask_scale=1, seed_mask=None):
    self.mask = mask
    self.seed_mask = seed_mask
    self._shift_mask_scale = shift_mask_scale
    self.shift_mask = None
    if shift_mask is not None:
      self.shift_mask = np.max(np.abs(shift_mask), axis=0) >= shift_mask_threshold
      assert shift_mask_fov is not None
      # the box is given in (x, y, z); start may be negative
      self._shift_mask_fov_pre_offset = np.asarray(shift_mask_fov.start)[::-1]
      self._shift_mask_fov_post_offset = np.asarray(shift_mask_fov.end)[::-1] - 1

  def is_valid_seed(self, pos):
    return not (self.seed_mask is not None and self.seed_mask[tuple(pos)])

  def is_valid_pos(self, pos):
    if self.mask is not None and self.mask[tuple(pos)]:
      return False
    if self.shift_mask is not None:
      np_pos = np.array(pos)
      fov_low = np.maximum(np_pos + self._shift_mask_fov_pre_offset, 0)
      fov_high = np_pos + self._shift_mask_fov_post_offset
      start = fov_low // self._shift_mask_scale
      end = fov_high // self._shift_mask_scale
      # z is a section index (not scaled), y / x are in shift-mask pixels (movement.py:323-331)
      if np.any(self.shift_mask[fov_low[0]:fov_high[0] + 1, start[1]:end[1] + 1, start[2]:end[2] + 1]):
        return False
    return True

  def movement_mask(self, shape):
    """Boolean [Z, Y, X]: True where `is_valid_pos` is False (None when nothing is restricted)."""
    shape = tuple(int(v) for v in shape)
    blocked = None if self.mask is None else np.asarray(self.mask).astype(bool)
    if self.shift_mask is None:
      return blocked
    sm = np.asarray(self.shift_mask)
    # summed-area table with a zero border: box sums for every position from eight gathers
    sat = np.zeros(tuple(d + 1 for d in sm.shape), dtype=np.int64)
    sat[1:, 1:, 1:] = sm.astype(np.int64).cumsum(0).cumsum(1).cumsum(2)
    bounds = []
    for axis in range(3):
      scale = 1 if axis == 0 else self._shift_mask_scale
      pre, post = int(self._shift_mask_fov_pre_offset[axis]), int(self._shift_mask_fov_post_offset[axis])
      lo = np.empty(shape[axis], dtype=np.int64)
      hi = np.empty(shape[axis], dtype=np.int64)
      for p in range(shape[axis]):
        first = max(p + pre, 0)
        last = p + post
        if axis:
          first, last = first // scale, last // scale
        b, e, _ = slice(first, last + 1).indices(sm.shape[axis])     # numpy's clipping, negative stops included
        lo[p], hi[p] = b, max(e, b)
      bounds.append((lo, hi))
    (z0, z1), (y0, y1), (x0, x1) = bounds

    def corner(zi, yi, xi):
      return sat[np.ix_(zi, yi, xi)]
    total = (corner(z1, y1, x1) - corner(z0, y1, x1) - corner(z1, y0, x1) - corner(z1, y1, x0) +
             corner(z0, y0, x1) + corner(z0, y1, x0) + corner(z1, y0, x0) - corner(z0, y0, x0))
    shifted = total > 0
    return shifted if blocked is None else (blocked | shifted)
