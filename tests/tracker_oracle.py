"""numpy restatement of the reference's EvalTracker as examples.py feeds it (ffn/training/tracker.py, examples.py), on
top of the example-loop oracle.  It is pinned against the reference's own tracker by tests/golden/tracker_ref.npz
(tests/golden/make_golden_tracker.py), and the device tracker (ffn_examples_tracker) is pinned against it.

What it keeps: the moves record_move counts (fixed_offsets: every evaluated target at int(|shift|); max_pred_offsets:
every popped entry inside max_radius and in an unvisited cell, at radius 0), and for every finished example add_patch's
prediction counts at logit(0.9), its eval voxels, its mean loss in float64 and its centre planes in a 16-deep ring.
"""

import collections

import numpy as np
from scipy import special

import examples_oracle as eo
from ffn_b200.training import examples as ex
from ffn_b200.training import tracker as tk

SUMMARY_EVERY = 10   # the fixture takes get_summaries() and reset() after every 10th step

# Deliberate bugs; each changes the comparison with the fixture in at least one case:
BUGS = (
    'radius_round',       # the move radius rounded instead of truncated
    'max_pred_radius',    # max_pred_offsets' moves counted at their own radius instead of 0
    'skipped_recorded',   # queue entries skipped as outside max_radius or visited counted (as missed moves)
    'eval_gt',            # seed > logit(0.9) written against a Python float, i.e. '>' against the float32-rounded
                          # value under NEP 50 (a float64 '>' equals '>=' on float32 logits: logit(0.9) is no float32)
    'no_eval_crop',       # add_patch on the whole max_pred_moves patch instead of its eval crop
)


class TrackerOracle(eo.ExampleLoopOracle):

  def __init__(self, *args, bugs=(), **kw):
    super().__init__(*args, **kw)
    assert set(bugs) <= set(BUGS), bugs
    self.bugs = set(bugs)
    fov_moves = self.moves - (1 if self.policy == 'max_pred_moves' else 0)
    self.eval = np.array(tk.eval_shape(self.fov, self.deltas, fov_moves))
    self.radii = tk.radii(ex.model_shifts(self.deltas) + list(self.shifts))
    self.entries = {}
    self.reset()

  def reset(self):
    self.steps = self.patches = self.eval_voxels = 0
    self.pred = np.zeros(4, np.int64)
    self.loss = 0.0
    self.loss_mag = 0.0   # sum over patches of mean(max(x, 0) + |x z| + log1p(exp(-|x|))): the loss's error scale
    self.moves_r = {r: np.zeros(3, np.int64) for r in self.radii}
    self.ring = collections.deque(maxlen=tk.RING)

  # --- EvalTracker.record_move ------------------------------------------------------------------------------------
  def record_move(self, wanted, executed, off):
    n = float(np.linalg.norm(np.asarray(off, np.float64)))
    r = int(round(n)) if 'radius_round' in self.bugs else int(n)
    m = self.moves_r.setdefault(r, np.zeros(3, np.int64))
    if wanted:
      m[0 if executed else 1] += 1
    elif executed:
      m[2] += 1

  # --- the policies, recording as examples.py does, and add_patch when exhausted (get_example) ----------------------
  def load(self, entry):
    self.entries[self.loaded] = (int(entry['volume']), tuple(int(v) for v in entry['center_xyz']))
    return super().load(entry)

  def _fixed(self, el):
    for off in [(0, 0, 0)] + self.shifts:
      valid, wanted = self._eval(el['seed'], el['labels'], off)
      self.record_move(wanted, valid, off)
      if valid:
        yield off
    self.add_patch(el)

  def _max_pred(self, el):
    queue = collections.deque([(0, 0, 0)])
    done = set()
    d = self.deltas
    while queue:
      off = np.array(queue.popleft())
      if np.any(np.abs(off) > self.max_radius):
        if 'skipped_recorded' in self.bugs:
          self.record_move(True, False, (0, 0, 0))
        continue
      q = tuple(int(v) for v in (2 * off + d) // (2 * np.maximum(d, 1)))
      if q in done:
        if 'skipped_recorded' in self.bugs:
          self.record_move(True, False, (0, 0, 0))
        continue
      valid, wanted = self._eval(el['seed'], el['labels'], tuple(off))
      self.record_move(wanted, valid, tuple(off) if 'max_pred_radius' in self.bugs else (0, 0, 0))
      if not valid or (not wanted and q != (0, 0, 0)):
        continue
      done.add(q)
      yield tuple(int(v) for v in off)
      todos = sorted(self._scored_moves(el['seed'], off), reverse=True)
      queue.extend(tuple(int(v) for v in off + np.array(p)) for _, p in todos)
    self.add_patch(el)

  # --- EvalTracker.add_patch --------------------------------------------------------------------------------------
  def add_patch(self, el):
    shape = self.size if 'no_eval_crop' in self.bugs else self.eval
    start = self.size // 2 - shape // 2
    win = tuple(slice(s, s + n) for s, n in zip(start, shape))
    logits, labels = el['seed'][win], el['labels'][win]
    x, z = logits.astype(np.float64), labels.astype(np.float64)
    soft = np.log1p(np.exp(-np.abs(x)))
    self.loss += float(np.sum(np.maximum(x, 0.0) - x * z + soft)) / x.size
    self.loss_mag += float(np.sum(np.maximum(x, 0.0) + np.abs(x * z) + soft)) / x.size
    pred = logits > float(tk.EVAL_THRESHOLD) if 'eval_gt' in self.bugs else logits >= tk.EVAL_THRESHOLD
    true = labels > 0.5
    self.pred += [np.sum(pred & true), np.sum(~pred & ~true), np.sum(pred & ~true), np.sum(~pred & true)]
    self.eval_voxels += labels.size
    self.patches += 1
    c = shape // 2
    planes = tuple((labels[i], logits[i]) for i in (np.s_[c[0], :, :], np.s_[:, c[1], :], np.s_[:, :, c[2]]))
    self.ring.append((planes, self.entries.pop(el['example'])))

  def next(self, entries):
    out = super().next(entries)
    self.steps += 1
    return out

  def state(self, reset=False):
    s = tk.TrackerState(steps=self.steps, fov_voxels=self.steps * self.batch * int(np.prod(self.fov)),
                        patches=self.patches, eval_voxels=self.eval_voxels, prediction_counts=self.pred.copy(),
                        patch_loss=self.loss, moves={r: m.copy() for r, m in self.moves_r.items()},
                        planes=[p for p, _ in self.ring], coords=[c for _, c in self.ring])
    if reset:
      self.reset()
    return s


def make(c, bugs=()):
  return TrackerOracle(c['volumes'], c['offset_scale'], c['fov'], c['deltas'], c['batch'], c['policy'],
                       c['fov_moves'], ex.seed_logits(0.05), ex.thresholds(c['threshold']), c['shifts'], bugs=bugs)


def eval_snapped_logits(rng, batch, fov_zyx):
  """float32(logit(0.9)), which lies above the float64 eval threshold, the float32 below it (below the threshold),
  and a low value: both sides of the eval threshold, exactly at its float32 neighbours."""
  hi = np.float32(tk.EVAL_THRESHOLD)
  assert float(hi) > tk.EVAL_THRESHOLD
  lo = np.nextafter(hi, np.float32(-np.inf))
  vals = np.array([hi, lo, hi - 6], np.float32)
  return vals[rng.choice(3, size=(batch,) + tuple(fov_zyx), p=[0.3, 0.3, 0.4])]


def step_logits(rng, c):
  if c['snap'] == 'eval':
    return eval_snapped_logits(rng, c['batch'], c['fov'])
  if c['snap'] == 'low':   # every shift fails: every example finishes one step after it starts
    return np.full((c['batch'],) + tuple(c['fov']), -3.0, np.float32)
  return eo.step_logits(rng, c)


def cases():
  """examples_oracle's ten cases, and three of the tracker's own: the eval threshold's float32 neighbours under both
  policies (at threshold 0.9 the move threshold is the same logit), and 20 elements that all finish every step, more
  than the 16 ring slots."""
  return eo.cases() + [
      ('fixed_eval_snap', (7, 7, 7), (2, 2, 2), 'fixed', 1, 0.9, 3, (1, 2), (0, 1, 2), 2, 21, 'eval'),
      ('max_pred_eval_snap', (7, 7, 7), (2, 2, 2), 'max_pred_moves', 1, 0.9, 2, (1, 2), (0,), 2, 22, 'eval'),
      ('fixed_batch20', (5, 5, 5), (1, 1, 1), 'fixed', 1, 0.9, 20, (), (0,), 1, 23, 'low'),
  ]


def ref_summaries(c, state):
  """Scalars by tag of tracker.summaries on an oracle reading (images left out)."""
  return {t: v for t, v in tk.summaries(state, ['vol%d' % i for i in range(len(c['volumes']))], images=False)}
