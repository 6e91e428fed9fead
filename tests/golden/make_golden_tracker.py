"""Tracker fixture: the REAL reference `ffn/training/tracker.py` (EvalTracker), fed by its unmodified `examples.py`,
`mask.py` and `inference/movement.py`, driven as train.py:353-423 drives them.

    python tests/golden/make_golden_tracker.py

The loop is make_golden_examples.py's (its `reference_modules()`, serial executor and `load_example`), with the
reference's own EvalTracker passed where that script passes a stub.  What the tracker is given besides:
  * tracker.py does not compile as shipped: the `try:` of slice_image (tracker.py:235) has an empty body.  It is
    compiled in memory with that body set to `raise IOError`, so that it takes its `except` branch, the
    `PIL.ImageFont.load_default()` font;
  * stand-ins for TensorFlow, by TF's documented semantics, for the calls of the eager path only:
    `executing_eagerly()` is True; `reduce_mean` is a float32 mean; `nn.sigmoid_cross_entropy_with_logits` is
    max(x, 0) - x z + log1p(exp(-|x|)) in float32; `Summary.Value` / `Summary.Image` are plain records; the dtypes
    carry `as_numpy_dtype`;
  * `variables.TFSyncVariable` is the local-value plumbing only: `from_tf` reads the local value (this loop never
    calls to_tf, so the local value is what the TF variable would hold), and `reset` zeroes it.

Per case and step: the cumulative counters (moves, moves_<r>, prediction_counts, num_voxels, num_patches, loss,
fov_stats).  After every 10th step, get_summaries() then reset(), as train.py:415-423 does: every scalar by tag, and the decoded
RGB pixels of every image of the first summary (the images of all four would quadruple the file).  Output: tracker_ref.npz.
"""
import io
import os
import sys
import types

import numpy as np
from scipy import special

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as mg  # noqa: E402
import make_golden_examples as mge  # noqa: E402
import examples_oracle as eo  # noqa: E402
import tracker_oracle as to  # noqa: E402
from ffn_b200.training import examples as ex  # noqa: E402

OUT = os.path.join(HERE, 'tracker_ref.npz')


class _Record:
  def __init__(self, **kw):
    self.__dict__.update(kw)


class _SyncVariable:
  def __init__(self, name, shape, dtype):
    self._value = np.zeros(shape, dtype=dtype.as_numpy_dtype)
    self.tf_value = None

  @property
  def value(self):
    return self._value

  @property
  def from_tf(self):
    return self._value.copy()

  def reset(self):
    self._value = np.zeros_like(self._value)


def _sigmoid_xent(logits, labels):
  x = np.asarray(logits, np.float32)
  z = np.asarray(labels, np.float32)
  return np.maximum(x, np.float32(0)) - x * z + np.log1p(np.exp(-np.abs(x)))


def reference_tracker():
  """The reference's tracker module, compiled with the one repair, on the TensorFlow stand-ins."""
  tf = sys.modules['tensorflow.compat.v1']
  tf.executing_eagerly = lambda: True
  tf.reduce_mean = lambda x: np.mean(np.asarray(x, np.float32), dtype=np.float32)
  tf.nn = types.SimpleNamespace(sigmoid_cross_entropy_with_logits=_sigmoid_xent)
  tf.Summary = types.SimpleNamespace(Value=_Record, Image=_Record)
  tf.int64 = types.SimpleNamespace(as_numpy_dtype=np.int64)
  tf.float32 = types.SimpleNamespace(as_numpy_dtype=np.float32)
  variables = types.ModuleType('ffn.training.variables')
  variables.TFSyncVariable = _SyncVariable
  path = os.path.join(mg.REF, 'ffn', 'training', 'tracker.py')
  with open(path) as f:
    src = f.read()
  broken = '    try:\n\n      # font = PIL.ImageFont.load_default()\n    except (IOError, ValueError):'
  assert src.count(broken) == 1, 'tracker.py changed: the repair no longer applies'
  src = src.replace(broken, '    try:\n      raise IOError\n    except (IOError, ValueError):')
  mod = types.ModuleType('ffn.training.tracker_ref')
  mod.__package__ = 'ffn.training'
  mod.__file__ = path
  exec(compile(src, path, 'exec'), mod.__dict__)  # pylint: disable=exec-used
  mod.variables = variables   # `from . import variables` finds the package's real module, already imported
  return mod


def _counters(t):
  out = {'moves': t.moves.value.copy(), 'prediction_counts': t.prediction_counts.value.copy(),
         'num_voxels': t.num_voxels.value.copy(), 'num_patches': t.num_patches.value.copy(),
         'loss': t.loss.value.copy(), 'fov_stats': t.fov_stats.value.copy()}
  for r, v in t.moves_by_r.items():
    out['moves_r=%d' % r] = v.value.copy()
  return out


def run_reference(examples, inputs, tracker_mod, c):
  """make_golden_examples.run_reference's loop with the reference's EvalTracker."""
  B = c['batch']
  mge._Serial.batch, mge._Serial.submitted = B, 0
  size_xyz = list(c['size'][::-1])
  names = ['vol%d' % i for i in range(len(c['volumes']))]
  image_map = {n: v[0] for n, v in zip(names, c['volumes'])}
  label_map = {n: v[1] for n, v in zip(names, c['volumes'])}
  state = {'next': 0}

  def load_example():
    row = c['rows'][state['next']]
    state['next'] += 1
    coord = np.array([row[1:4]], np.int64)
    vname = np.array([names[row[0]].encode('ascii')])
    labels = np.asarray(inputs.load_from_numpylike(coord, vname, size_xyz, label_map))
    patch = np.asarray(inputs.load_from_numpylike(coord, vname, size_xyz, image_map))
    radii = np.array(size_xyz) // 2
    lom = (labels > 0) & (labels == labels[0, radii[2], radii[1], radii[0], 0])
    labels = np.where(lom, np.float32(0.95), np.float32(0.05)).astype(np.float32)
    full = [0] + [1 + int(p) for p in row[4:7]] + [4]
    refl = tuple(1 + a for a in range(3) if row[7 + a])
    labels, patch = np.transpose(labels, full), np.transpose(patch, full)
    if refl:
      labels, patch = np.flip(labels, refl), np.flip(patch, refl)
    off, scale = c['offset_scale'][row[0]]
    patch = (patch.astype(np.float32) - off) / scale
    return patch, labels, np.ones_like(labels), coord, vname

  thr = special.logit(c['threshold'])
  if c['policy'] == 'fixed':
    inner = lambda info, seed, labels, t: examples.fixed_offsets(  # noqa: E731
        info, seed, labels, t, thr, fov_shifts=[tuple(s[::-1]) for s in c['shifts'].tolist()])
  else:
    moves = c['fov_moves'] + 1
    inner = lambda info, seed, labels, t: examples.max_pred_offsets(  # noqa: E731
        info, seed, labels, t, thr, max_radius=np.array(c['deltas'][::-1]) * moves)

  eval_zyx = [f + 2 * d * c['fov_moves'] for f, d in zip(c['fov'], c['deltas'])]   # train.py:167-169
  model_shifts_xyz = [s[::-1] for s in ex.model_shifts(c['deltas'])]
  tracker = tracker_mod.EvalTracker(eval_zyx, model_shifts_xyz)
  tracker.sess = types.SimpleNamespace(run=lambda ops, feed=None: list(ops))
  info = types.SimpleNamespace(deltas=list(c['deltas'][::-1]), input_seed_size=list(c['fov'][::-1]),
                               input_image_size=list(c['fov'][::-1]), pred_mask_size=list(c['fov'][::-1]))
  it = examples.BatchExampleIter(
      lambda: examples.get_example(load_example, tracker, info, inner, np.float32(0.05), seed_shape=tuple(c['size'])),
      tracker, B, info)
  rng = np.random.RandomState(c['logit_seed'])
  steps, summaries = [], []
  for step in range(eo.N_STEPS):
    next(it)
    it.update_seeds(to.step_logits(rng, c)[..., None])
    steps.append(_counters(tracker))
    if (step + 1) % to.SUMMARY_EVERY == 0:
      scalars, images = {}, {}
      for v in tracker.get_summaries():
        if getattr(v, 'image', None) is not None:
          import PIL.Image  # pylint: disable=g-import-not-at-top
          im = np.asarray(PIL.Image.open(io.BytesIO(v.image.encoded_image_string)).convert('RGB'))
          assert im.shape == (v.image.height, v.image.width, 3)
          images[v.tag] = im
        else:
          scalars[v.tag] = float(v.simple_value)
      summaries.append((step, scalars, images))
      tracker.reset()
  return steps, summaries


def main():
  examples, inputs = mge.reference_modules()
  tracker_mod = reference_tracker()
  out = {'n_cases': len(to.cases()), 'n_steps': eo.N_STEPS}
  for i, case in enumerate(to.cases()):
    c = eo.case_setup(case)
    steps, summaries = run_reference(examples, inputs, tracker_mod, c)
    for k in steps[0]:
      out['c%d/%s' % (i, k)] = np.stack([s[k] for s in steps])
    for step, scalars, images in summaries:
      p = 'c%d/s%d/' % (i, step)
      out[p + 'tags'] = np.array(sorted(scalars))
      out[p + 'values'] = np.array([scalars[t] for t in sorted(scalars)], np.float64)
      if step == to.SUMMARY_EVERY - 1:   # images of the first summary only, to keep the fixture small
        for tag, im in images.items():
          out[p + tag] = im
    last = steps[-1]
    print('%-20s patches %s, moves %s, prediction counts %s, %d summaries' % (
        c['tag'], sum(int(s['num_patches'][0]) for s in steps[9::10]), last['moves'], last['prediction_counts'],
        len(summaries)))
  np.savez_compressed(OUT, **out)
  print('wrote %s (%d bytes)' % (OUT, os.path.getsize(OUT)))


if __name__ == '__main__':
  main()
