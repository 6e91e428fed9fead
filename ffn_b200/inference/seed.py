"""Seed policies: iterators over (z, y, x) starting points, computed once per canvas.

Mirrors ffn/inference/seed.py: `BaseSeedPolicy` (:37-130, incl. the border filter :81-88 and the
checkpoint state :100-113), `PolicyPeaks` (:142-199), `PolicyPeaks2d` (:202-280), `PolicyFillEmptySpace`
(:283-304), `PolicyMax` (:307-313), `PolicyMaxPeaks` (:316-352), `PolicyGrid3d` (:411-430), `PolicyGrid2d`
(:433-452), `PolicyInvertOrigins` (:455-469), `PolicyDenseSeeds` (:472-492), `ReverseCoords` (:495-504),
`SequentialPolicies` (:507-544).  `PolicyImagePeaks3D2D` and `PolicyImagePeaks2DDisk` are not provided: they
add no tie-break noise, so their output on real images depends on how skimage orders and spaces equal-valued
peaks.

`PolicyPeaks`, `PolicyPeaks2d`, `PolicyFillEmptySpace` and `PolicyMaxPeaks` run on the device when the canvas
has one (the image, segmentation and masks are resident there; only the RandomState(42) tie-break noise is
uploaded), and otherwise with scipy on the host; both paths yield the same list.  PolicyPeaks2d / FillEmptySpace
define one case the reference leaves to the `edt` package: with no finite distance (a slice without an edge
voxel, a canvas without a labelled voxel) there are no seeds.

`PolicyPeaks` depends upstream on `edt.edt` and `skimage.feature.peak_local_max`, neither of
which is installable offline; it is restated with scipy (exact Euclidean distance transform with
anisotropy, maximum-filter peak detection with the same seeded tie-break noise).  Seed ORDER and
the tie-break follow the reference; exact equality with skimage's peak suppression is not
guaranteed (SURVEY.md 8c), which is why flood-fill parity always feeds both sides the same list.
"""

import weakref

import numpy as np
from scipy import ndimage

from . import storage


class BaseSeedPolicy:
  """Base class: subclasses fill `self.coords` ([N, 3] zyx) in `init_coords`."""

  def __init__(self, canvas, **kwargs):
    del kwargs
    self.canvas = weakref.proxy(canvas)
    self.coords = None
    self.idx = 0

  def init_coords(self):
    raise NotImplementedError()

  def __iter__(self):
    return self

  def _ensure_coords(self):
    """Runs init_coords once and applies the border filter (seed.py:76-88)."""
    if self.coords is None:
      self.init_coords()
      if self.coords is None:
        return False
      self.coords = np.asarray(self.coords).reshape(-1, 3)
      if self.coords.size:
        margin = np.array(self.canvas.margin)[np.newaxis, ...]
        keep = np.all((self.coords - margin >= 0) & (self.coords + margin < self.canvas.shape), axis=1)
        self.coords = self.coords[keep, :]
    return True

  def __next__(self):
    if not self._ensure_coords():
      raise StopIteration()
    if self.idx < self.coords.shape[0]:
      curr = self.coords[self.idx, :]
      self.idx += 1
      return tuple(int(v) for v in curr)
    raise StopIteration()

  def next(self):
    return self.__next__()

  def remaining(self):
    """All not-yet-consumed seeds as an [N, 3] array (what the device loop is given)."""
    if not self._ensure_coords():
      return np.zeros((0, 3), dtype=np.int32)
    return np.ascontiguousarray(self.coords[self.idx:], dtype=np.int32)

  def get_state(self, previous=False):
    if previous:
      return self.coords, max(0, self.idx - 1)
    return self.coords, self.idx

  def set_state(self, state):
    self.coords, self.idx = state

  def get_exclusion_mask(self):
    mask = np.asarray(self.canvas.segmentation) > 0
    if self.canvas.restrictor is not None:
      if self.canvas.restrictor.mask is not None:
        mask |= self.canvas.restrictor.mask
      if self.canvas.restrictor.seed_mask is not None:
        mask |= self.canvas.restrictor.seed_mask
    return mask


_NOISE_CACHE = {}


def _tie_break_noise(shape):
  """RandomState(42).rand(*shape) (seed.py:133-139), cached for the most recent shape: a run over many
  equally sized subvolumes draws the same 8 bytes / voxel every time (0.7 s for 512^3)."""
  if shape not in _NOISE_CACHE:
    _NOISE_CACHE.clear()
    _NOISE_CACHE[shape] = np.random.RandomState(seed=42).rand(*shape)
  return _NOISE_CACHE[shape]


class PolicyPeaks(BaseSeedPolicy):
  """Sobel edges -> adaptive threshold -> distance transform -> local maxima (seed.py:142-199)."""

  def init_coords(self):
    dev = getattr(self.canvas, '_dev', None)
    restrictor = self.canvas.restrictor
    # The device's movement mask also carries the shift-mask rule, which seed.py:170-173 does not apply
    # to the edge map: with a shift mask the seeds are computed by the host restatement below.
    if dev is not None and getattr(restrictor, 'shift_mask', None) is None:
      # device path: the canvas' image / segmentation / masks are already resident in HBM
      noise = _tie_break_noise(tuple(int(v) for v in self.canvas.shape))
      with self.canvas._exec_client.engine_lock:         # pylint: disable=protected-access
        self.coords = dev.seed_peaks(self.canvas.voxel_size_zyx, noise).astype(np.int64).reshape(-1, 3)
      return
    # host path (shift masks / no device canvas): the same stages with scipy
    blocked = self._blocked_voxels()
    is_edge = _edge_mask(np.asarray(self.canvas.image), blocked)
    if is_edge.all():
      return
    dist = _distance_map(is_edge, self.canvas.voxel_size_zyx, self.get_exclusion_mask())
    noise = _tie_break_noise(tuple(int(v) for v in self.canvas.shape))
    # peak_local_max(min_distance=3, threshold_abs=0, threshold_rel=0) with its default exclude_border=True:
    # peaks closer than 3 voxels to the canvas border are dropped (seed.py:191)
    peaks = _local_peaks(dist + noise * 1e-4, 3, 0, 0)
    self.coords = np.array(sorted(map(tuple, peaks.astype(int).tolist()))).reshape(-1, 3)

  def _blocked_voxels(self):
    """Voxels the restrictor forbids (movement mask | seed mask), or None."""
    r = self.canvas.restrictor
    parts = [m for m in (getattr(r, 'mask', None), getattr(r, 'seed_mask', None)) if m is not None]
    if not parts:
      return None
    out = np.zeros(self.canvas.shape, dtype=bool)
    for m in parts:
      out |= np.asarray(m).astype(bool)
    return out


def _edge_mask(image, blocked):
  """Sobel gradient magnitude above its local (gaussian, sigma 49/6) average; blocked voxels count as edges so that
  large masked regions do not distort the distance transform (seed.py:152-173)."""
  grad = ndimage.generic_gradient_magnitude(image.astype(np.float32), ndimage.sobel)
  local = np.empty_like(grad)
  ndimage.gaussian_filter(grad, 49.0 / 6.0, output=local, mode='reflect')
  out = grad > local
  if blocked is not None:
    out |= blocked
  return out


def _distance_map(is_edge, voxel_size_zyx, excluded):
  """Distance (physical units) to the nearest edge, -1 where seeds are not allowed (seed.py:183-188)."""
  dist = ndimage.distance_transform_edt(~is_edge, sampling=voxel_size_zyx).astype(np.float32)
  dist[excluded | ~np.isfinite(dist)] = -1
  return dist


def _device_canvas(canvas, uses_movement_mask):
  """The canvas' DeviceCanvas when a policy may run there, else None.  The device's movement mask also
  carries the shift-mask rule, which the reference's policies do not apply: a policy that reads
  `restrictor.mask` runs on the host when a shift mask is set."""
  dev = getattr(canvas, '_dev', None)
  if dev is not None and uses_movement_mask and getattr(canvas.restrictor, 'shift_mask', None) is not None:
    return None
  return dev


def _local_peaks(keys, min_distance, threshold_abs, threshold_rel):
  """skimage.feature.peak_local_max(keys, min_distance, threshold_abs, threshold_rel) by its documented
  definition: a voxel is a peak iff it equals the maximum of its (2 min_distance + 1)^ndim neighbourhood
  (edges clamped), exceeds max(threshold_abs, threshold_rel * max) (threshold_abs None: the minimum) and lies
  at least min_distance from the border on every axis.  Non-finite keys are never peaks and do not enter the
  minimum / maximum.  Returns the peak indices in C order."""
  finite = np.isfinite(keys)
  if not finite.any():
    return np.zeros((0, keys.ndim), dtype=np.int64)
  thr = float(keys[finite].min()) if threshold_abs is None else float(threshold_abs)
  if threshold_rel is not None:
    thr = max(thr, float(threshold_rel) * float(keys[finite].max()))
  size = 2 * min_distance + 1
  peak = (keys == ndimage.maximum_filter(keys, size=size, mode='nearest')) & (keys > thr) & finite
  inner = np.zeros(keys.shape, dtype=bool)
  inner[tuple(slice(min_distance, s - min_distance) for s in keys.shape)] = True
  return np.argwhere(peak & inner)


class PolicyPeaks2d(BaseSeedPolicy):
  """Per z-slice: 2-D Sobel edges -> adaptive threshold -> 2-D distance transform -> local maxima
  (seed.py:202-280).  Only the movement mask counts as edges; seeds in labelled or seed-masked voxels are
  proposed and rejected later by the canvas, as in the reference.  A slice without any edge voxel has no
  finite distance and yields no seeds."""

  def __init__(self, canvas, min_distance=7, threshold_abs=2.5, sort_cmp='ascending', **kwargs):
    super().__init__(canvas, **kwargs)
    self.min_distance = min_distance
    self.threshold_abs = threshold_abs
    self.sort_reverse = sort_cmp.strip().lower().startswith('de')

  def init_coords(self):
    shape = tuple(int(v) for v in self.canvas.shape)
    noise = _tie_break_noise(shape[1:])     # every slice draws the same RandomState(42) plane
    dev = _device_canvas(self.canvas, uses_movement_mask=True)
    if dev is not None:
      with self.canvas._exec_client.engine_lock:         # pylint: disable=protected-access
        coords = dev.seed_policy('peaks_2d', self.min_distance, self.threshold_abs, 0, noise)
    else:
      image = np.asarray(self.canvas.image)
      mask = getattr(self.canvas.restrictor, 'mask', None)
      chunks = []
      for z in range(shape[0]):
        is_edge = _edge_mask(image[z], None)
        if mask is not None:
          is_edge |= np.asarray(mask[z]).astype(bool)
        if not is_edge.any():
          continue
        dt = ndimage.distance_transform_edt(~is_edge).astype(np.float32)
        idx = _local_peaks(dt + noise * 1e-4, self.min_distance, self.threshold_abs, 0)
        chunks.append(np.concatenate([np.full((idx.shape[0], 1), z, dtype=np.int64), idx], axis=1))
      coords = np.concatenate(chunks, axis=0) if chunks else np.zeros((0, 3), dtype=np.int64)
    self.coords = np.array(sorted(map(tuple, np.asarray(coords).astype(int).tolist()),
                                  reverse=self.sort_reverse)).reshape(-1, 3)


class PolicyFillEmptySpace(BaseSeedPolicy):
  """Local maxima of the distance transform of the unlabelled voxels (seed.py:283-304): seeds for the gaps
  of an existing segmentation (init_segmentation, or an earlier policy of SequentialPolicies).  The -1
  markers count as labelled.  A canvas without any labelled voxel yields no seeds."""

  def init_coords(self):
    shape = tuple(int(v) for v in self.canvas.shape)
    noise = _tie_break_noise(shape)
    dev = _device_canvas(self.canvas, uses_movement_mask=False)
    if dev is not None:
      with self.canvas._exec_client.engine_lock:         # pylint: disable=protected-access
        coords = dev.seed_policy('fill_empty', 2, 0.5, 0, noise)
    else:
      empty = np.asarray(self.canvas.segmentation) == 0
      if empty.all():
        coords = np.zeros((0, 3), dtype=np.int64)
      else:
        dt = ndimage.distance_transform_edt(empty).astype(np.float32)
        coords = _local_peaks(dt + noise * 1e-4, 2, 0.5, 0)
    self.coords = np.array(sorted(map(tuple, np.asarray(coords).astype(int).tolist()))).reshape(-1, 3)


class PolicyMaxPeaks(BaseSeedPolicy):
  """Local maxima of the image intensity with the excluded voxels (labels, movement mask, seed mask) set to 0
  (seed.py:316-352)."""

  def __init__(self, canvas, min_distance=3, threshold_abs=0, threshold_rel=0, **kwargs):
    super().__init__(canvas, **kwargs)
    self.min_distance = min_distance
    self.threshold_abs = threshold_abs
    self.threshold_rel = threshold_rel

  def init_coords(self):
    shape = tuple(int(v) for v in self.canvas.shape)
    noise = _tie_break_noise(shape)
    dev = _device_canvas(self.canvas, uses_movement_mask=True)
    if dev is not None:
      with self.canvas._exec_client.engine_lock:         # pylint: disable=protected-access
        coords = dev.seed_policy('max_peaks', self.min_distance, self.threshold_abs, self.threshold_rel, noise)
    else:
      img = np.asarray(self.canvas.image).astype(np.float32)
      img[self.get_exclusion_mask()] = 0
      coords = _local_peaks(img + noise * 1e-4, self.min_distance, self.threshold_abs, self.threshold_rel)
    self.coords = np.array(sorted(map(tuple, np.asarray(coords).astype(int).tolist()))).reshape(-1, 3)


class PolicyMax(BaseSeedPolicy):
  """All voxels in descending order of intensity (seed.py:307-313)."""

  def init_coords(self):
    image = np.asarray(self.canvas.image)
    order = np.argsort(image.ravel())[::-1]
    self.coords = np.stack(np.unravel_index(order, image.shape), axis=1)


class PolicyGrid3d(BaseSeedPolicy):
  """Uniform 3d grid visited offset by offset (seed.py:411-430)."""

  def __init__(self, canvas, step=16, offsets=(0, 8, 4, 12, 2, 10, 14), **kwargs):
    super().__init__(canvas, **kwargs)
    self.step = step
    self.offsets = offsets

  def init_coords(self):
    shape = self.canvas.shape
    coords = []
    for offset in self.offsets:
      for z in range(offset, shape[0], self.step):
        for y in range(offset, shape[1], self.step):
          for x in range(offset, shape[2], self.step):
            coords.append((z, y, x))
    self.coords = np.array(coords).reshape(-1, 3)


class PolicyGrid2d(BaseSeedPolicy):
  """Uniform 2d grid on every z plane (seed.py:433-452)."""

  def __init__(self, canvas, step=16, offsets=(0, 8, 4, 12, 2, 6, 10, 14), **kwargs):
    super().__init__(canvas, **kwargs)
    self.step = step
    self.offsets = offsets

  def init_coords(self):
    shape = self.canvas.shape
    coords = []
    for offset in self.offsets:
      for z in range(shape[0]):
        for y in range(offset, shape[1], self.step):
          for x in range(offset, shape[2], self.step):
            coords.append((z, y, x))
    self.coords = np.array(coords).reshape(-1, 3)


class PolicyInvertOrigins(BaseSeedPolicy):
  """Seeds of a previous run in reverse id order (seed.py:455-469)."""

  def __init__(self, canvas, corner=None, segmentation_dir=None, **kwargs):
    super().__init__(canvas, **kwargs)
    self.corner = corner
    self.segmentation_dir = segmentation_dir

  def init_coords(self):
    origins = storage.load_origins(self.segmentation_dir, self.corner)
    points = sorted(origins.items(), reverse=True)
    self.coords = np.array([info.start_zyx for _, info in points]).reshape(-1, 3)


class PolicyDenseSeeds(BaseSeedPolicy):
  """Every voxel above a threshold, after optional erosions (seed.py:472-492)."""

  def __init__(self, canvas, threshold=0.5, num_erosions=0, invert=False, **kwargs):
    super().__init__(canvas, **kwargs)
    self._threshold = threshold
    self._num_erosions = num_erosions
    self._invert = invert

  def init_coords(self):
    x = np.asarray(self.canvas.image) > self._threshold
    if self._invert:
      x = ~x
    for _ in range(self._num_erosions):
      # skimage.morphology.binary_erosion (seed.py:488): connectivity-1 cross, outside of the image counts as foreground
      x = ndimage.binary_erosion(x, border_value=True)
    self.coords = np.array(np.where(x)).T


class ReverseCoords(BaseSeedPolicy):
  """Wraps another policy and reverses its order (seed.py:495-504)."""

  def __init__(self, canvas, policy_to_reverse, **policy_kwargs):
    super().__init__(canvas)
    self._policy = globals()[policy_to_reverse](canvas, **policy_kwargs)

  def init_coords(self):
    self.coords = np.array(list(self._policy)[::-1]).reshape(-1, 3)


class SequentialPolicies(BaseSeedPolicy):
  """Runs several policies one after another (seed.py:507-544)."""

  def __init__(self, canvas, policies, **kwargs):
    super().__init__(canvas, **kwargs)
    self._policies = [globals()[name](canvas, **dict(args, **kwargs)) for name, args in policies]

  def init_coords(self):
    chunks = [np.array(list(p)).reshape(-1, 3) for p in self._policies]
    self.coords = np.concatenate(chunks, axis=0) if chunks else np.zeros((0, 3), dtype=np.int64)
