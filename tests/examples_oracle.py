"""numpy restatement of the training example loop (ffn_b200/training/examples.py, ffn_b200/csrc/examples.cu).

It restates the reference's train.py:202-286 (load, object mask, soften, PermuteAndReflect, normalise) and
ffn/training/examples.py (get_example, BatchExampleIter, fixed_offsets, max_pred_offsets with
movement.get_scored_move_offsets), with the two choices the device makes where the reference does not: new examples
go to the elements in element order, and they come from an explicit stream of FfnExampleCoord entries.  It is pinned
against the reference's own examples.py by tests/golden/examples_ref.npz, and the device is pinned against it.
"""

import collections

import numpy as np

from ffn_b200 import _lib
from ffn_b200.training import examples as ex

N_STEPS = 40
FULL_STEPS = (0, 7, N_STEPS - 1)


class ExampleLoopOracle:
  """volumes: [(uint8 image, int64 labels)], offset_scale: [(float32 offset, float32 scale)], per volume index."""

  def __init__(self, volumes, offset_scale, fov_zyx, deltas_zyx, batch, fov_policy='fixed', fov_moves=1,
               seed_logits=(np.float32(-2.944439), np.float32(2.944439)), thresholds=(2.1972245773362196, 0.9),
               shifts_zyx=(), f32=()):
    """f32: deliberate bugs for the tests, a subset of {'valid', 'wanted', 'score'}: that comparison is made against
    the float32-rounded threshold instead of in float64."""
    self.volumes = volumes
    self.offset_scale = [(np.float32(o), np.float32(s)) for o, s in offset_scale]
    self.fov = np.array(fov_zyx)
    self.deltas = np.array(deltas_zyx)
    self.batch = batch
    self.policy = fov_policy
    self.moves = fov_moves + 1 if fov_policy == 'max_pred_moves' else fov_moves
    self.size = self.fov + 2 * self.deltas * self.moves
    self.pad_logit, self.centre_logit = np.float32(seed_logits[0]), np.float32(seed_logits[1])
    # np.float64, as scipy returns them: a float32 value compared with them is promoted (NEP 50 would compare a
    # float32 with a Python float in float32)
    self.seed_thr, self.label_thr = np.float64(thresholds[0]), np.float64(thresholds[1])
    self.thr = {k: np.float32(self.label_thr if k == 'wanted' else self.seed_thr) if k in f32 else
                (self.label_thr if k == 'wanted' else self.seed_thr) for k in ('valid', 'wanted', 'score')}
    self.shifts = [tuple(int(v) for v in s) for s in shifts_zyx]
    self.max_radius = self.deltas * self.moves
    self.elements = [None] * batch   # (image, labels, seed, generator, example index, offset)
    self.loaded = 0

  # --- loading (train.py:202-286) ---------------------------------------------------------------------------------
  def load(self, entry):
    image_vol, label_vol = self.volumes[int(entry['volume'])]
    start = np.array(entry['center_xyz'][::-1], np.int64) - (self.size - 1) // 2
    sl = tuple(slice(s, s + n) for s, n in zip(start, self.size))
    assert (start >= 0).all() and all(s.stop <= n for s, n in zip(sl, label_vol.shape))
    labels = label_vol[sl].astype(np.int64)
    image = image_vol[sl]
    centre = labels[tuple(self.size // 2)]
    lom = (labels > 0) & (labels == centre)
    labels = np.where(lom, np.float32(0.95), np.float32(0.05)).astype(np.float32)
    perm = [int(p) for p in entry['permutation_zyx']]
    refl = tuple(d for d in range(3) if entry['reflect_zyx'][d])
    labels = np.transpose(labels, perm)
    image = np.transpose(image, perm)
    if refl:
      labels = np.flip(labels, refl)
      image = np.flip(image, refl)
    off, scale = self.offset_scale[int(entry['volume'])]
    image = ((image.astype(np.float32) - off) / scale).astype(np.float32)
    seed = np.full(tuple(self.size), self.pad_logit, np.float32)
    seed[tuple(self.size // 2)] = self.centre_logit
    return np.ascontiguousarray(image), np.ascontiguousarray(labels), seed

  # --- move policies (examples.py:159-198, 286-328) --------------------------------------------------------------
  def _eval(self, seed, labels, off):
    c = tuple(self.size // 2 + np.array(off))
    return seed[c] >= self.thr['valid'], labels[c] >= self.thr['wanted']

  def _fixed(self, el):
    for off in [(0, 0, 0)] + self.shifts:
      valid, _ = self._eval(el['seed'], el['labels'], off)
      if valid:
        yield off

  def _scored_moves(self, seed, off):
    """movement.get_scored_move_offsets on the fov crop of the seed at off, (score, (z, y, x)) tuples."""
    start = self.size // 2 - self.fov // 2 + np.array(off)
    crop = seed[tuple(slice(s, s + n) for s, n in zip(start, self.fov))]
    centre = np.array(crop.shape) // 2
    sub = [slice(c - d, c + d + 1) for c, d in zip(centre, self.deltas)]
    out, done = [], set()
    for axis, d in enumerate(self.deltas):
      if d == 0:
        continue
      for ao in (-d, d):
        sel = sub[:]
        sel[axis] = ao + centre[axis]
        face = crop[tuple(sel)]
        pos = np.unravel_index(face.argmax(), face.shape)
        score = face[pos]
        if score < self.thr['score']:
          continue
        rel = [int(pos[0] - face.shape[0] // 2), int(pos[1] - face.shape[1] // 2)]
        rel.insert(axis, int(ao))
        r = (score, tuple(rel))
        if r not in done:
          done.add(r)
          out.append(r)
    return out

  def _max_pred(self, el):
    queue = collections.deque([(0, 0, 0)])
    done = set()
    d = self.deltas
    while queue:
      off = np.array(queue.popleft())
      if np.any(np.abs(off) > self.max_radius):
        continue
      q = tuple(int(v) for v in (2 * off + d) // (2 * np.maximum(d, 1)))
      if q in done:
        continue
      valid, wanted = self._eval(el['seed'], el['labels'], tuple(off))
      if not valid or (not wanted and q != (0, 0, 0)):
        continue
      done.add(q)
      yield tuple(int(v) for v in off)
      todos = sorted(self._scored_moves(el['seed'], off), reverse=True)
      queue.extend(tuple(int(v) for v in off + np.array(p)) for _, p in todos)

  # --- the loop (get_example, BatchExampleIter) -------------------------------------------------------------------
  def next(self, entries):
    """One step: (seed, image, labels [batch, F], offsets [batch, 3], example indices [batch], entries taken)."""
    taken = 0
    for e in range(self.batch):
      el = self.elements[e]
      off = next(el['gen'], None) if el is not None else None
      if off is None:
        image, labels, seed = self.load(entries[taken])
        el = {'image': image, 'labels': labels, 'seed': seed, 'example': self.loaded}
        el['gen'] = self._fixed(el) if self.policy == 'fixed' else self._max_pred(el)
        self.loaded += 1
        taken += 1
        off = next(el['gen'])
        assert off == (0, 0, 0)
        self.elements[e] = el
      el['off'] = off
    crops = [np.stack([self._crop(el[k], el['off']) for el in self.elements]) for k in ('seed', 'image', 'labels')]
    offsets = np.array([el['off'] for el in self.elements], np.int32)
    example = np.array([el['example'] for el in self.elements], np.int64)
    return crops[0], crops[1], crops[2], offsets, example, taken

  def _window(self, off):
    start = self.size // 2 - self.fov // 2 + np.array(off)
    return tuple(slice(s, s + n) for s, n in zip(start, self.fov))

  def _crop(self, a, off):
    return a[self._window(off)]

  def update(self, logits):
    for el, lg in zip(self.elements, logits):
      el['seed'][self._window(el['off'])] = lg

  def seeds(self):
    return np.stack([el['seed'] for el in self.elements])


def fake_logits(rng, batch, fov_zyx, scale=4.0, bias=1.5):
  """Seeded float32 logits spread around the move threshold, so that moves both pass and fail."""
  return (rng.standard_normal((batch,) + tuple(fov_zyx)) * scale + bias).astype(np.float32)


def snapped_logits(rng, batch, fov_zyx, seed_threshold):
  """Seeded float32 logits of three values: the largest float32 below the float64 seed threshold (it fails in
  float64, but passes against the threshold rounded to float32 when that rounds down), the smallest one above it
  (rare, so that a face's maximum is often the one below), and a low value."""
  t = np.float64(seed_threshold)
  lo = np.float32(t)
  if lo >= t:
    lo = np.nextafter(lo, np.float32(-np.inf))
  hi = np.nextafter(lo, np.float32(np.inf))
  vals = np.array([lo, hi, t - 4.0], np.float32)
  return vals[rng.choice(3, size=(batch,) + tuple(fov_zyx), p=[0.35, 0.03, 0.62])]


def step_logits(rng, c):
  """The logits the fixture and the tests paste after every step of case c."""
  if c['snap']:
    return snapped_logits(rng, c['batch'], c['fov'], ex.thresholds(c['threshold'])[0])
  return fake_logits(rng, c['batch'], c['fov'])


def model_shifts_shuffled(deltas_zyx, rng):
  """model.shifts in a seeded order, as train.py's random.shuffle leaves them (zero deltas give duplicates)."""
  s = ex.model_shifts(deltas_zyx)
  return [s[i] for i in rng.permutation(len(s))]


# --- the fixture's cases (tests/golden/make_golden_examples.py), regenerated from their seeds by the tests --------------
def cases():
  """(tag, fov zyx, deltas zyx, policy, fov_moves, threshold, batch, permutable, reflectable, n volumes, seed,
  snapped logits).

  The snapped cases put logits one float32 step either side of the float64 seed threshold, at thresholds whose
  float32 rounding lies below them (0.9499999, 0.7): a move, or a face maximum, of the value below is refused in
  float64 and taken in float32.  At 0.0500000023 the label threshold rounds to 0.05f in float32 but lies above it, so
  background labels are unwanted in float64 and wanted in float32.  A face maximum just below the threshold is queued
  only under a float32 test; it changes the path when a later paste makes its voxel valid before it is popped, which
  the small faces and long runs of max_pred_scores provoke."""
  return [
      ('fixed', (7, 7, 7), (2, 2, 2), 'fixed', 1, 0.9, 4, (1, 2), (0, 1, 2), 2, 1, False),
      ('fixed_zero_delta', (5, 7, 7), (0, 2, 2), 'fixed', 1, 0.9499999, 3, (1, 2), (), 1, 2, False),
      ('fixed_moves2', (7, 7, 7), (1, 2, 2), 'fixed', 2, 0.9, 2, (), (0, 2), 2, 3, False),
      ('max_pred', (7, 7, 7), (2, 2, 2), 'max_pred_moves', 1, 0.9, 4, (0, 1, 2), (0, 1, 2), 2, 4, False),
      ('max_pred_aniso', (5, 7, 9), (2, 1, 0), 'max_pred_moves', 2, 0.9499999, 2, (), (1,), 1, 5, False),
      ('max_pred_wide', (9, 9, 9), (3, 3, 3), 'max_pred_moves', 1, 0.9, 1, (1, 2), (2,), 3, 6, False),
      ('fixed_snapped', (7, 7, 7), (2, 2, 2), 'fixed', 1, 0.9499999, 3, (1, 2), (0, 1, 2), 1, 7, True),
      ('max_pred_snapped', (7, 7, 7), (2, 2, 2), 'max_pred_moves', 1, 0.7, 2, (), (0,), 1, 8, True),
      ('max_pred_labels', (7, 7, 7), (2, 2, 1), 'max_pred_moves', 1, 0.0500000023, 3, (), (), 2, 9, True),
      ('max_pred_scores', (7, 7, 7), (1, 2, 2), 'max_pred_moves', 2, 0.7, 2, (), (0,), 1, 11, True),
  ]


def volumes(rng, n, shape):
  """Blocky signed labels (negative ids and 0 are background) and uint8 images, with per-volume offset and scale."""
  out = []
  for _ in range(n):
    idx = [np.cumsum(rng.rand(s) < 0.3) for s in shape]
    ids = np.array([0, 3, -2, 5, 7, 0, 9, -6, 11, 12], np.int64)
    lab = ids[(idx[0][:, None, None] * 5 + idx[1][None, :, None] * 3 + idx[2][None, None, :]) % len(ids)]
    img = rng.randint(0, 256, shape).astype(np.uint8)
    out.append((img, np.ascontiguousarray(lab)))
  return out


def stream(rng, n, vols, size, permutable, reflectable):
  """n FfnExampleCoord entries (int32 [n, 10]) whose crops of `size` (z, y, x) lie inside their volumes."""
  out = np.zeros((n, 10), np.int32)
  for i in range(n):
    v = rng.randint(len(vols))
    shape = vols[v][1].shape
    c = [rng.randint((s - 1) // 2, n_ - s + (s - 1) // 2 + 1) for s, n_ in zip(size, shape)]
    perm = np.arange(3)
    if permutable:
      perm[list(permutable)] = np.array(permutable)[rng.permutation(len(permutable))]
    refl = np.zeros(3, np.int32)
    for a in reflectable:
      refl[a] = rng.rand() > 0.5
    out[i] = [v] + c[::-1] + list(perm) + list(refl)
  return out


def as_coords(rows):
  out = np.zeros(len(rows), _lib.EXAMPLE_COORD_DTYPE)
  out['volume'] = rows[:, 0]
  out['center_xyz'] = rows[:, 1:4]
  out['permutation_zyx'] = rows[:, 4:7]
  out['reflect_zyx'] = rows[:, 7:10]
  return out


def case_setup(case):
  tag, fov, deltas, policy, moves, thr, batch, perm, refl, nvol, seed, snap = case
  rng = np.random.RandomState(seed)
  m = moves + 1 if policy == 'max_pred_moves' else moves
  size = tuple(f + 2 * d * m for f, d in zip(fov, deltas))
  vols = volumes(rng, nvol, tuple(s + 6 + 2 * k for k, s in enumerate(size)))
  offset_scale = [(np.float32(rng.uniform(90, 160)), np.float32(rng.uniform(20, 60))) for _ in range(nvol)]
  rows = stream(rng, N_STEPS * batch, vols, size, perm, refl)
  shifts = model_shifts_shuffled(deltas, rng) if policy == 'fixed' else []
  return dict(tag=tag, fov=fov, deltas=deltas, policy=policy, fov_moves=moves, threshold=thr, batch=batch,
              permutable=perm, reflectable=refl, size=size, volumes=vols, offset_scale=offset_scale, rows=rows,
              shifts=np.array(shifts, np.int32).reshape(-1, 3), logit_seed=1000 * seed, snap=snap)


