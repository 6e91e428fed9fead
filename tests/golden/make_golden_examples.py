"""Training-example fixture: the REAL reference `ffn/training/examples.py`, `mask.py` and `inference/movement.py`,
unmodified, driven as train.py:353-412 drives them.

    python tests/golden/make_golden_examples.py

Third-party imports are stubbed by make_golden.install_stubs().  What the reference is given besides, and nothing else:
  * `examples.futures.ThreadPoolExecutor` is a serial executor, so the element generators advance in element order
    (the order the device defines) instead of racing in a thread pool;
  * `tracker.EvalTracker` is a stub that records nothing;
  * `load_example` reads the volumes through `inputs.load_from_numpylike`'s own inner loader (a `tf.py_func` stub calls
    it, with a `BoundingBox` that has connectomics' `to_slice3d`), then applies train.py:251-274's TF ops restated
    in numpy: the object mask of the centre label, soften_labels, PermuteAndReflect (`np.transpose`, `np.flip`) and
    offset_and_scale_patches in float32.  The examples come from an explicit stream: volume index, centre (x, y, z),
    permutation and reflections of each;
  * the logits of every step are seeded float32 noise around the move threshold, or, in the snapped cases, values
    one float32 step either side of the float64 threshold (examples_oracle.step_logits).

Per case and step: every element's offset (z, y, x, recorded from the policy generator's yields) and example index,
and the full batch (seed, image, labels) at a few steps.  Output: examples_ref.npz.
"""
import functools
import os
import sys
import types

import numpy as np
from scipy import special

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as mg  # noqa: E402
import examples_oracle as eo  # noqa: E402

OUT = os.path.join(HERE, 'examples_ref.npz')
from examples_oracle import N_STEPS, FULL_STEPS, case_setup, cases  # noqa: E402


class _Serial:
  """concurrent.futures.ThreadPoolExecutor, run in the caller's thread in submission order."""
  submitted = 0

  def __init__(self, max_workers=None):
    pass

  def __enter__(self):
    return self

  def __exit__(self, *a):
    return False

  def submit(self, fn, *args):
    _Serial.current = _Serial.submitted % _Serial.batch
    _Serial.submitted += 1
    r = fn(*args)
    return types.SimpleNamespace(result=lambda: r)


class _Tracker:
  def __getattr__(self, name):
    return lambda *a, **k: None


class _BBox:
  def __init__(self, start, size):
    self.start, self.size = np.asarray(start), np.asarray(size)

  def to_slice3d(self):
    e = self.start + self.size
    return np.index_exp[self.start[2]:e[2], self.start[1]:e[1], self.start[0]:e[0]]


class _Loaded(np.ndarray):
  def set_shape(self, shape):
    assert list(self.shape) == list(shape), (self.shape, shape)


def reference_modules():
  mg.install_stubs()
  sys.path.insert(0, mg.REF)
  tracker = types.ModuleType('ffn.training.tracker')
  tracker.EvalTracker = _Tracker
  sys.modules['ffn.training.tracker'] = tracker
  sys.modules['connectomics.common.bounding_box'].BoundingBox = _BBox
  # inputs.py imports augmentation.py, whose TF-only transforms are restated in numpy here
  sys.modules['ffn.training.augmentation'] = mg._Stub('ffn.training.augmentation')
  from ffn.training import examples, inputs, mask  # noqa: F401
  from ffn.inference import movement  # noqa: F401
  import ffn
  assert os.path.dirname(ffn.__file__).startswith(mg.REF), ffn.__file__
  examples.futures = types.SimpleNamespace(ThreadPoolExecutor=_Serial)

  class _NameScope:
    def __init__(self, *a):
      pass

    def __enter__(self):
      return 'scope'

    def __exit__(self, *a):
      return False

  inputs.tf = types.SimpleNamespace(name_scope=_NameScope, squeeze=lambda x, axis: x[axis],
                                    py_func=lambda f, args, dtypes, name=None: [f(*args).view(_Loaded)])
  return examples, inputs


def run_reference(examples, inputs, c):
  B = c['batch']
  _Serial.batch, _Serial.submitted = B, 0
  size_xyz = list(c['size'][::-1])
  names = ['vol%d' % i for i in range(len(c['volumes']))]
  image_map = {n: v[0] for n, v in zip(names, c['volumes'])}
  label_map = {n: v[1] for n, v in zip(names, c['volumes'])}
  state = {'next': 0}
  example_idx = np.full(B, -1, np.int64)
  last_off = np.zeros((B, 3), np.int32)

  def load_example():
    row = c['rows'][state['next']]
    example_idx[_Serial.current] = state['next']
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
    inner = functools.partial(examples.fixed_offsets, fov_shifts=[tuple(s[::-1]) for s in c['shifts'].tolist()],
                              threshold=thr)
  else:
    moves = c['fov_moves'] + 1
    inner = functools.partial(examples.max_pred_offsets, max_radius=np.array(c['deltas'][::-1]) * moves,
                              threshold=thr)

  def policy(info, seed, labels, tracker):
    for off in inner(info, seed, labels, tracker):
      last_off[_Serial.current] = off[::-1]
      yield off

  info = types.SimpleNamespace(deltas=list(c['deltas'][::-1]), input_seed_size=list(c['fov'][::-1]),
                               input_image_size=list(c['fov'][::-1]), pred_mask_size=list(c['fov'][::-1]))
  pad = np.float32(0.05)
  it = examples.BatchExampleIter(
      lambda: examples.get_example(load_example, _Tracker(), info, policy, pad, seed_shape=tuple(c['size'])),
      _Tracker(), B, info)
  rng = np.random.RandomState(c['logit_seed'])
  out = {'offsets': [], 'example': [], 'consumed': []}
  for step in range(N_STEPS):
    before = state['next']
    seed, image, labels, _ = next(it)
    out['offsets'].append(last_off.copy())
    out['example'].append(example_idx.copy())
    out['consumed'].append(state['next'] - before)
    if step in FULL_STEPS:
      for k, v in (('seed', seed), ('image', image), ('labels', labels)):
        out['%s_%d' % (k, step)] = v[..., 0]
    it.update_seeds(eo.step_logits(rng, c)[..., None])
  return out


def main():
  examples, inputs = reference_modules()
  out = {'n_cases': len(cases()), 'n_steps': N_STEPS, 'full_steps': np.array(FULL_STEPS)}
  for i, case in enumerate(cases()):
    c = case_setup(case)
    r = run_reference(examples, inputs, c)
    loads = int(np.sum(r['consumed']))
    print('%-18s %d examples loaded, %d distinct offsets' % (c['tag'], loads,
                                                             len(set(map(tuple, np.concatenate(r['offsets']))))))
    out['offsets_%d' % i] = np.array(r['offsets'], np.int32)
    out['example_%d' % i] = np.array(r['example'], np.int64)
    out['consumed_%d' % i] = np.array(r['consumed'], np.int64)
    for s in FULL_STEPS:
      for k in ('seed', 'image', 'labels'):
        out['%s_%d_%d' % (k, i, s)] = r['%s_%d' % (k, s)]
  np.savez_compressed(OUT, **out)
  print('wrote %s (%d bytes)' % (OUT, os.path.getsize(OUT)))


if __name__ == '__main__':
  main()
