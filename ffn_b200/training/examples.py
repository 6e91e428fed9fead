"""The training example loop of the reference's train.py on the device (ffn_examples_* of include/ffn_b200.h).

`ExampleLoop` holds, per batch element, a training patch loaded from a training coordinate (train.py:202-286), its
seed canvas and the state of its field-of-view move policy (ffn/training/examples.py: `fixed_offsets` or
`max_pred_offsets`).  `Trainer.train(loop, n)` runs n training steps fed by it with no host copy between them.

Two things are defined here where the reference leaves them to TensorFlow or to a thread race:
  * the example stream: every record of the coordinate files, permuted per epoch with
    `np.random.RandomState(seed)`, with each example's axis permutation and reflections drawn from the same stream
    (the reference's `shuffle_batch` and PermuteAndReflect draws cannot be reproduced without TensorFlow; the
    distribution is the same);
  * which element takes which new example: the elements in order 0 .. batch-1 within a step (the reference's
    element generators load examples from a thread pool).
"""

from __future__ import annotations

import ctypes as C
from typing import Mapping, Sequence

import numpy as np
from scipy import special

from .. import _lib
from . import tracker as _tracker

LABEL_SOFT_TRUE = np.float32(0.95)


def model_shifts(deltas_zyx) -> list[tuple[int, int, int]]:
  """ConvStack3DFFNModel.shifts (model.py:75-81) as (z, y, x) offsets, in the reference's order.  With a zero delta
  the list holds duplicates, which the fixed policy visits as the reference does."""
  dz, dy, dx = (int(v) for v in deltas_zyx)
  out = []
  for x in (-dx, 0, dx):
    for y in (-dy, 0, dy):
      for z in (-dz, 0, dz):
        if x == 0 and y == 0 and z == 0:
          continue
        out.append((z, y, x))
  return out


def patch_moves(fov_policy: str, fov_moves: int) -> int:
  """train.py's fov_moves(): one more move for max_pred_moves."""
  return fov_moves + 1 if fov_policy == 'max_pred_moves' else fov_moves


def seed_logits(seed_pad: float) -> tuple[np.float32, np.float32]:
  """special.logit(mask.make_seed(..., pad=seed_pad)) in float32: (the pad value, the centre value)."""
  v = special.logit(np.array([seed_pad, 0.95], np.float32))
  return np.float32(v[0]), np.float32(v[1])


def thresholds(threshold: float) -> tuple[float, float]:
  """(logit(threshold), expit(logit(threshold))) in float64: the seed and label thresholds of a move."""
  t = float(special.logit(threshold))
  return t, float(special.expit(t))


class ExampleStream:
  """The seeded example stream: records permuted per epoch, a permutation of the permutable axes and a reflection
  decision per reflectable axis drawn per example, all from one `np.random.RandomState(seed)`."""

  def __init__(self, volume_index: np.ndarray, centers_xyz: np.ndarray, permutable_zyx=(), reflectable_zyx=(),
               seed: int = 0):
    self.volume_index = np.asarray(volume_index, np.int32)
    self.centers_xyz = np.asarray(centers_xyz, np.int32).reshape(-1, 3)
    if len(self.volume_index) != len(self.centers_xyz) or not len(self.centers_xyz):
      raise ValueError('the stream needs one volume index per centre, and at least one record')
    self.permutable = np.array(sorted(int(a) for a in permutable_zyx), np.int64)
    self.reflectable = np.array(sorted(int(a) for a in reflectable_zyx), np.int64)
    self.rng = np.random.RandomState(seed)
    self._order = np.empty(0, np.int64)
    self._pos = 0

  def take(self, n: int) -> np.ndarray:
    out = np.zeros(n, _lib.EXAMPLE_COORD_DTYPE)
    for i in range(n):
      if self._pos == len(self._order):
        self._order = self.rng.permutation(len(self.centers_xyz))
        self._pos = 0
      r = self._order[self._pos]
      self._pos += 1
      perm = np.arange(3, dtype=np.int32)
      if self.permutable.size:
        perm[self.permutable] = self.permutable[self.rng.permutation(self.permutable.size)]
      refl = np.zeros(3, np.int32)
      if self.reflectable.size:
        refl[self.reflectable] = self.rng.random_sample(self.reflectable.size) > 0.5
      out[i] = (self.volume_index[r], self.centers_xyz[r], perm, refl)
    return out

  def get_state(self) -> dict:
    """The position in the stream: the generator's MT19937 state, this epoch's order and the position in it, as
    numpy values."""
    _, keys, pos, has_gauss, gauss = self.rng.get_state()
    return {'rng_keys': np.array(keys, np.uint32), 'rng_pos': np.int64(pos), 'rng_has_gauss': np.int64(has_gauss),
            'rng_gauss': np.float64(gauss), 'order': self._order.copy(), 'pos': np.int64(self._pos)}

  def set_state(self, state: Mapping[str, np.ndarray]):
    """Continues the stream where `get_state` left it.  A state that does not fit this stream's records is refused
    (ValueError), changing nothing."""
    n = len(self.centers_xyz)
    order = np.asarray(state['order'], np.int64).reshape(-1)
    pos = int(state['pos'])
    if len(order) not in (0, n) or (len(order) and not np.array_equal(np.sort(order), np.arange(n))):
      raise ValueError('the stream state\'s epoch order is not a permutation of this stream\'s %d records' % n)
    if not 0 <= pos <= len(order):
      raise ValueError('the stream state\'s position %d lies outside its epoch of %d records' % (pos, len(order)))
    rng = np.random.RandomState()
    rng.set_state(('MT19937', np.asarray(state['rng_keys'], np.uint32), int(state['rng_pos']),
                   int(state['rng_has_gauss']), float(state['rng_gauss'])))
    self.rng, self._order, self._pos = rng, order, pos


def _image_volume(v, name):
  v = np.asarray(v)
  if v.dtype != np.uint8:
    raise TypeError('image volume %r must be uint8, got %s' % (name, v.dtype))
  if v.ndim != 3:
    raise ValueError('image volume %r must be 3-d (single channel), got shape %r' % (name, v.shape))
  return np.ascontiguousarray(v)


def _label_volume(v, name):
  v = np.asarray(v)
  if v.ndim != 3:
    raise ValueError('label volume %r must be 3-d, got shape %r' % (name, v.shape))
  if v.dtype.kind not in 'iub' or v.dtype == np.bool_:
    raise TypeError('label volume %r must hold integers, got %s' % (name, v.dtype))
  if v.dtype.kind == 'u' and v.dtype.itemsize == 8 and v.size and int(v.max()) >= 2**63:
    raise ValueError('label volume %r holds ids at or above 2^63, which int64 labels cannot hold' % (name,))
  return np.ascontiguousarray(v, dtype=np.int64)


class ExampleLoop:
  """Per batch element: the training patch, the seed canvas and the move policy's state, on one GPU.

  volumes: {name: (uint8 image [z, y, x], integer labels [z, y, x])}.  offset_scale: {name: (offset, scale)}, with
  (image_mean, image_stddev) for the other names.  stream: an ExampleStream over the same names' indices (in the
  order of `names`).  shifts_zyx: the fixed policy's visiting order after the centre (default: model_shifts)."""

  def __init__(self, volumes: Mapping[str, tuple[np.ndarray, np.ndarray]], stream: ExampleStream,
               fov_zyx=(33, 33, 33), deltas_zyx=(8, 8, 8), batch_size: int = 4, fov_policy: str = 'fixed',
               fov_moves: int = 1, seed_pad: float = 0.05, threshold: float = 0.9, shifts_zyx=None,
               offset_scale: Mapping[str, tuple[float, float]] | None = None, image_mean=None, image_stddev=None,
               device: int = 0):
    if fov_policy not in _lib.FOV_POLICIES:
      raise ValueError('unknown fov_policy %r (fixed and max_pred_moves are supported)' % (fov_policy,))
    if not 0.0 < float(threshold) < 1.0:
      raise ValueError('threshold must lie in (0, 1), got %r' % (threshold,))
    offset_scale = dict(offset_scale or {})
    self.names = list(volumes)
    self._lib = _lib.load()
    self.fov_zyx = tuple(int(v) for v in fov_zyx)
    self.deltas_zyx = tuple(int(v) for v in deltas_zyx)
    self.batch_size = int(batch_size)
    self.moves = patch_moves(fov_policy, int(fov_moves))
    self.patch_zyx = tuple(f + 2 * d * self.moves for f, d in zip(self.fov_zyx, self.deltas_zyx))
    self.stream = stream
    self._pending = np.zeros(0, _lib.EXAMPLE_COORD_DTYPE)
    self.consumed = 0

    keep, vols = [], []
    for name in self.names:
      image, labels = volumes[name]
      image, labels = _image_volume(image, name), _label_volume(labels, name)
      if name in offset_scale:
        off, scale = offset_scale[name]
      elif image_mean is None or image_stddev is None:
        raise ValueError('no offset and scale for volume %r: give image_mean and image_stddev or an '
                         'offset_scale entry' % (name,))
      else:
        off, scale = image_mean, image_stddev
      keep += [image, labels]
      vols.append(_lib.ExampleVolume(image=image.ctypes.data, labels=labels.ctypes.data,
                                     image_shape_zyx=_lib.i3(image.shape), label_shape_zyx=_lib.i3(labels.shape),
                                     offset=float(np.float32(off)), scale=float(np.float32(scale))))
    vol_arr = (_lib.ExampleVolume * len(vols))(*vols)
    shifts = np.ascontiguousarray(model_shifts(self.deltas_zyx) if shifts_zyx is None else shifts_zyx,
                                  np.int32).reshape(-1, 3)
    pad_logit, centre_logit = seed_logits(seed_pad)
    seed_thr, label_thr = thresholds(threshold)
    desc = _lib.ExampleDesc(policy=_lib.FOV_POLICIES[fov_policy], fov_moves=int(fov_moves), seed_pad=float(seed_pad),
                            seed_logit_pad=float(pad_logit), seed_logit_centre=float(centre_logit),
                            batch=self.batch_size, seed_threshold=seed_thr, label_threshold=label_thr,
                            shifts_zyx=shifts.ctypes.data, n_shifts=len(shifts),
                            eval_threshold=float(_tracker.EVAL_THRESHOLD))
    perm = set(int(a) for a in stream.permutable)
    refl = set(int(a) for a in stream.reflectable)
    desc.permutable_zyx = _lib.i3([int(a in perm) for a in range(3)])
    desc.reflectable_zyx = _lib.i3([int(a in refl) for a in range(3)])
    model = _lib.ModelDesc()
    model.fov_zyx = _lib.i3(self.fov_zyx)
    model.deltas_zyx = _lib.i3(self.deltas_zyx)
    model.depth = 1
    model.features = 32
    self.eval_zyx = _tracker.eval_shape(self.fov_zyx, self.deltas_zyx, fov_moves)
    # EvalTracker's radii come from model.shifts; the fixed policy's own shifts may add more
    self.radii = _tracker.radii(model_shifts(self.deltas_zyx) + (shifts.tolist() if fov_policy == 'fixed' else []))
    h = C.c_void_p()
    _lib.check(self._lib.ffn_examples_create(int(device), C.byref(model), C.byref(desc), C.cast(vol_arr, C.c_void_p),
                                             len(vols), C.byref(h)))
    self._h = h
    del keep

  @property
  def handle(self):
    if not getattr(self, '_h', None):
      raise RuntimeError('the example loop is closed')
    return self._h

  def close(self):
    if getattr(self, '_h', None):
      self._lib.ffn_examples_destroy(self._h)
      self._h = None

  def __del__(self):
    self.close()

  def entries(self, n: int) -> np.ndarray:
    """The next n unconsumed stream entries (drawn from the stream as needed)."""
    if len(self._pending) < n:
      self._pending = np.concatenate([self._pending, self.stream.take(n - len(self._pending))])
    return np.ascontiguousarray(self._pending[:n])

  def consume(self, n: int):
    self._pending = self._pending[n:]
    self.consumed += n

  def get_state(self) -> dict:
    """The loop's state: the device blob (ffn_examples_get_state: per element the patches, the seed, the move policy
    and the tracker), the stream entries drawn but not yet consumed and the count consumed.  Reads only; it may be
    taken between `next` and `update`.  The stream's own state is `stream.get_state()`."""
    return {'device': _lib.get_state(self._lib.ffn_examples_get_state, self.handle), 'pending': self._pending.copy(),
            'consumed': np.int64(self.consumed)}

  def set_state(self, state: Mapping[str, np.ndarray]):
    """Restores a `get_state` of a loop of the same geometry, thresholds, shifts and volumes.  A refused state
    (RuntimeError names the field that differs) changes nothing."""
    pending = np.asarray(state['pending'])
    if pending.dtype != _lib.EXAMPLE_COORD_DTYPE or pending.ndim != 1:
      raise ValueError('the loop state\'s pending entries are not a 1-d array of stream entries')
    _lib.set_state(self._lib.ffn_examples_set_state, self.handle, state['device'])
    self._pending = pending.copy()
    self.consumed = int(state['consumed'])

  def next(self):
    """One step of the loop: (seed, image, labels) [batch, Z, Y, X] float32, offsets [batch, 3] (z, y, x) from the
    patch centres, and each element's example index in the stream."""
    b = self.batch_size
    coords = self.entries(b)
    seed, image, labels = (np.empty((b,) + self.fov_zyx, np.float32) for _ in range(3))
    offsets = np.empty((b, 3), np.int32)
    example = np.empty(b, np.int64)
    n = C.c_int64()
    _lib.check(self._lib.ffn_examples_next(self.handle, _lib.ptr(coords), len(coords), _lib.ptr(seed), _lib.ptr(image),
                                           _lib.ptr(labels), _lib.ptr(offsets), _lib.ptr(example), C.byref(n)))
    self.consume(int(n.value))
    return seed, image, labels, offsets, example

  def update(self, logits):
    """Pastes the network's logits [batch, Z, Y, X] into the seeds at the current offsets."""
    lg = np.ascontiguousarray(logits, dtype=np.float32)
    if lg.shape != (self.batch_size,) + self.fov_zyx:
      raise ValueError('logits must be [%d, %d, %d, %d]' % ((self.batch_size,) + self.fov_zyx))
    _lib.check(self._lib.ffn_examples_update(self.handle, _lib.ptr(lg)))

  def seeds(self) -> np.ndarray:
    """The seed canvases, [batch, patch z, y, x] float32."""
    out = np.empty((self.batch_size,) + self.patch_zyx, np.float32)
    _lib.check(self._lib.ffn_examples_read_seeds(self.handle, _lib.ptr(out)))
    return out

  def tracker(self, reset: bool = False) -> _tracker.TrackerState:
    """The tracker's counts since the last reset and the planes of the last (up to 16) finished examples, oldest
    first; reset: then zero the counts and empty the ring, as EvalTracker.reset() after get_summaries()."""
    counts = _lib.TrackerCounts()
    n_r = max(self.radii) + 1
    moves = np.zeros((n_r, 3), np.int64)
    pf = 2 * (self.eval_zyx[1] * self.eval_zyx[2] + self.eval_zyx[0] * self.eval_zyx[2] +
              self.eval_zyx[0] * self.eval_zyx[1])
    planes = np.zeros((_tracker.RING, pf), np.float32)
    coords = np.zeros(_tracker.RING, _lib.EXAMPLE_COORD_DTYPE)
    n = C.c_int32()
    _lib.check(self._lib.ffn_examples_tracker(self.handle, C.byref(counts), _lib.ptr(moves), n_r, _lib.ptr(planes),
                                              _lib.ptr(coords), C.byref(n), int(bool(reset))))
    k = n.value
    return _tracker.TrackerState(
        steps=counts.steps, fov_voxels=counts.steps * self.batch_size * int(np.prod(self.fov_zyx)),
        patches=counts.patches, eval_voxels=counts.eval_voxels,
        prediction_counts=np.array(counts.prediction_counts[:], np.int64), patch_loss=counts.patch_loss,
        moves={r: moves[r].copy() for r in self.radii},
        planes=[_tracker.split_planes(planes[i], self.eval_zyx) for i in range(k)],
        coords=[(int(c['volume']), tuple(int(v) for v in c['center_xyz'])) for c in coords[:k]])
