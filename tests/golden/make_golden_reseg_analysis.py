"""Resegmentation-analysis fixture: the REAL reference `ffn/inference/resegmentation_analysis.py`, unmodified, scoring
result files against an original segmentation.

    python tests/golden/make_golden_reseg_analysis.py

The module imports google3 libraries that do not exist outside Google, and it predates numpy 1.24.  Everything it is
given in their place, and nothing else:
  * `gfile.Open` -> `open`;
  * `logging` -> the standard library's `logging`;
  * `storage` -> the reference's own ffn/inference/storage.py, third-party imports stubbed as in make_golden_storage.py
    (only its `dequantize_probability` is used);
  * `resegmentation_pb2` -> this package's runtime-built messages, where `EndpointSegmentationResult` (the module's
    spelling) is `EndpointResegmentationResult` (the .proto's);
  * `np.int = int` (removed from numpy in 1.24);
  * `np.load(f)` -> `np.load(f, allow_pickle=True)`, the default before numpy 1.16.3: result files store ragged
    start points and histories as object arrays;
  * `pywrapsegment_util.ComputeOverlapCounts(a, b)` -> `{(old, new): number of voxels i with a[i] == old and
    b[i] == new}`.

Cases: pair and endpoint points on a synthetic segmentation with ids up to and above 2^63 at voxel size (30, 8, 8),
with an analysis radius below the resegmentation radius, several attempts per object (ragged start points; the last
one counts), FoV moves inside and outside the analysis box, an empty resegmented object, one touching the box border,
one filling the whole box, old id 0 among the endpoint overlaps, one IncompleteResegmentationError and one
InvalidBaseSegmentatonError each; plus the pair and the endpoint result of the reseg_64 process_point run.
The segmentation reaches the module as a volume store whose `[0, z0:z1, y0:y1, x0:x1]` is [1, z, y, x], as the
module's `[...][0, ...]` expects.
Output: reseg_analysis_ref.npz — per case the result file's name and bytes, the parameters, and the expected
`SerializeToString(deterministic=True)` or the name of the expected exception.
"""
import importlib.util
import io
import logging
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

OUT = os.path.join(HERE, 'reseg_analysis_ref.npz')
RADIUS = (6, 10, 12)           # z, y, x
ANALYSIS = (4, 7, 8)
VOXEL = (30, 8, 8)
BIG = 2**63 + 12345


def reference_module():
  mg.install_stubs()
  sys.path.insert(0, mg.REF)
  from ffn.inference import storage as ref_storage
  sys.path.insert(0, mg.REPO)
  from ffn_b200.inference import resegmentation_pb2

  def compute_overlap_counts(a, b):
    pairs, counts = np.unique(np.stack([np.asarray(a, np.uint64), np.asarray(b, np.uint64)]), axis=1,
                              return_counts=True)
    return {(int(o), int(n)): int(c) for (o, n), c in zip(pairs.T, counts)}

  class _Numpy(types.ModuleType):
    int = int

    def __getattr__(self, name):
      return getattr(np, name)

    @staticmethod
    def load(f, **kw):
      kw.setdefault('allow_pickle', True)
      return np.load(f, **kw)

  pb2 = types.ModuleType('resegmentation_pb2')
  pb2.EndpointSegmentationResult = resegmentation_pb2.EndpointResegmentationResult
  pb2.PairResegmentationResult = resegmentation_pb2.PairResegmentationResult
  injected = {
      'google3.pyglib.gfile': types.SimpleNamespace(Open=open),
      'google3.pyglib.logging': logging,
      'google3.research.neuromancer.segmentation.ffn.resegmentation_pb2': pb2,
      'google3.research.neuromancer.segmentation.ffn.storage': ref_storage,
      'google3.research.neuromancer.segmentation.python.pywrapsegment_util':
          types.SimpleNamespace(ComputeOverlapCounts=compute_overlap_counts),
  }
  for full, mod in injected.items():
    parts = full.split('.')
    for i in range(1, len(parts)):
      sys.modules.setdefault('.'.join(parts[:i]), types.ModuleType('.'.join(parts[:i])))
    parent, child = full.rsplit('.', 1)
    setattr(sys.modules[parent], child, mod)
  spec = importlib.util.spec_from_file_location(
      'ref_resegmentation_analysis', os.path.join(mg.REF, 'ffn/inference/resegmentation_analysis.py'))
  ref = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(ref)
  ref.np = _Numpy('numpy')
  return ref


class VolumeStore:
  """A 4-d label volume indexed as the module indexes it: an integer channel index keeps its axis."""

  def __init__(self, arr):
    self.arr = arr

  def __getitem__(self, ind):
    return self.arr[(slice(ind[0], ind[0] + 1),) + tuple(ind[1:])]


def synthetic_volume():
  """[1, Z, Y, X] uint64 slabs and blobs; ids include 0 (background) and ids >= 2^63."""
  rng = np.random.RandomState(7)
  vol = np.zeros((40, 48, 56), dtype=np.uint64)
  vol[:, :, :28] = 11
  vol[:, :, 28:] = 12
  vol[:, 30:, 20:40] = BIG
  vol[5:15, 5:20, 5:50] = BIG + 1
  vol[rng.rand(*vol.shape) < 0.04] = 0
  vol[18:23, 20:28, 24:33] = 0
  return vol[np.newaxis]


def probs_from(mask, rng):
  """uint8 quantised probabilities: above 0.5 inside `mask`, below it outside, with 0 (NaN, unvisited) and 128
  (127.5 / 255, exactly 0.5) at random."""
  hi = rng.randint(129, 256, mask.shape)
  lo = rng.randint(1, 128, mask.shape)
  q = np.where(mask, hi, lo).astype(np.uint8)
  q[rng.rand(*mask.shape) < 0.05] = 0
  q[mask & (rng.rand(*mask.shape) < 0.02)] = 128
  return q


def as_object(items):
  out = np.empty(len(items), dtype=object)
  for k, it in enumerate(items):
    out[k] = it
  return out


def write_file(probs, deletes, histories, start_points):
  buf = io.BytesIO()
  np.savez_compressed(buf, probs=np.asarray(probs, dtype=np.uint8), deletes=deletes, histories=histories,
                      start_points=start_points)
  return buf.getvalue()


def box_of(vol, zyx, radius):
  z, y, x = zyx
  rz, ry, rx = radius
  return vol[0, z - rz:z + rz + 1, y - ry:y + ry + 1, x - rx:x + rx + 1]


def synthetic_cases(vol):
  rng = np.random.RandomState(11)
  cases = []
  rz, ry, rx = RADIUS

  def moves(n, inside_frac=0.6):
    lo = np.array(RADIUS) - np.array(ANALYSIS)
    hi = lo + 2 * np.array(ANALYSIS)
    inside = rng.rand(n) < inside_frac
    pts = np.where(inside[:, None], rng.randint(lo, hi + 1, (n, 3)), rng.randint(0, 2 * np.array(RADIUS) + 1, (n, 3)))
    if n:
      pts[0] = lo           # on the corners: inclusive bounds
      pts[-1] = hi
    return pts.astype(np.int32)

  def pair(name, a, b, zyx, masks, attempts=(1, 1), steps=(7, 5), threshold=0.5, voxel=VOXEL, analysis=ANALYSIS,
           filled=(False, False)):
    # a filled object has probability 254.5 / 255 everywhere in the resegmentation box: above any threshold used here
    probs = np.stack([np.full(m.shape, 255, np.uint8) if f else probs_from(m, rng) for m, f in zip(masks, filled)])
    dels = [rng.randint(0, 40, n).astype(np.int64) for n in steps]
    hist = [moves(n) for n in steps]
    starts = as_object([rng.randint(0, 2 * np.array(RADIUS) + 1, (k, 3)) for k in attempts])
    data = write_file(probs, as_object(dels) if steps[0] != steps[1] else np.stack(dels),
                      as_object(hist) if steps[0] != steps[1] else np.stack(hist), starts)
    z, y, x = zyx
    cases.append(dict(name='%d-%d_at_%d_%d_%d.npz' % (a, b, x, y, z), kind='pair', file=data, radius=RADIUS,
                      analysis=analysis, voxel=voxel, threshold=threshold, tag=name))

  def grow(m, k=1):
    out = m.copy()
    for _ in range(k):
      out[1:] |= out[:-1]; out[:-1] |= out[1:]
      out[:, 1:] |= out[:, :-1]; out[:, :-1] |= out[:, 1:]
      out[:, :, 1:] |= out[:, :, :-1]; out[:, :, :-1] |= out[:, :, 1:]
    return out

  zyx = (20, 24, 28)
  box = box_of(vol, zyx, RADIUS)
  # a merge-worthy pair: each object regrows into the other; three attempts for the first object, one for the second
  pair('pair_merge', 11, 12, zyx, [grow(box == 11, 2) | (box == 12), (box == 12) | grow(box == 11, 1)],
       attempts=(3, 1), steps=(9, 6))
  # the second object empty; the first touches the box border and stays in its own segment
  pair('pair_empty_border', 12, 11, zyx, [box == 12, np.zeros(box.shape, bool)], attempts=(2, 2), steps=(4, 4))
  # ids >= 2^63; the first object fills the whole box (no background voxel for its distance transform)
  zyx2 = (10, 20, 30)
  box2 = box_of(vol, zyx2, RADIUS)
  pair('pair_big_ids_full', BIG + 1, 11, zyx2, [np.ones(box2.shape, bool), grow(box2 == 11)], attempts=(1, 4),
       steps=(3, 8), threshold=0.6, filled=(True, False))
  # analysis radius == resegmentation radius, isotropic voxels, nothing recorded for one object's moves
  zyx3 = (30, 36, 30)
  box3 = box_of(vol, zyx3, RADIUS)
  pair('pair_full_analysis', BIG, 12, zyx3, [grow(box3 == BIG), box3 == 12], steps=(5, 0), voxel=(1, 1, 1),
       analysis=RADIUS)
  # IncompleteResegmentationError: one object only
  probs = probs_from(box == 11, rng)[np.newaxis]
  cases.append(dict(name='11-12_at_%d_%d_%d.npz' % (zyx[2], zyx[1], zyx[0]), kind='pair',
                    file=write_file(probs, np.zeros((1, 3), np.int64), np.zeros((1, 3, 3), np.int32),
                                    as_object([np.zeros((1, 3), np.int64), np.zeros((0, 3), np.int64)])),
                    radius=RADIUS, analysis=ANALYSIS, voxel=VOXEL, threshold=0.5, tag='pair_incomplete'))
  # InvalidBaseSegmentatonError: the second id is not in the analysis box
  pair('pair_invalid', 11, 999, zyx, [box == 11, box == 12])

  def endpoint(name, a, zyx, mask, threshold=0.5):
    probs = probs_from(mask, rng)[np.newaxis]
    data = write_file(probs, np.zeros((1, 4), np.int64), np.zeros((1, 4, 3), np.int32),
                      as_object([np.array([[rz, ry, rx]]), np.zeros((0, 3), np.int64)]))
    z, y, x = zyx
    cases.append(dict(name='%d-0_at_%d_%d_%d.npz' % (a, x, y, z), kind='endpoint', file=data, radius=RADIUS,
                      analysis=ANALYSIS, voxel=VOXEL, threshold=threshold, tag=name))

  # the object spills over background (id 0) and its neighbours
  endpoint('endpoint_spill', 11, zyx, grow(box == 11, 2))
  endpoint('endpoint_big_ids', BIG + 1, zyx2, grow(box2 == BIG + 1) & (box2 != 11), threshold=0.7)
  endpoint('endpoint_empty', 12, zyx, np.zeros(box.shape, bool))
  endpoint('endpoint_invalid', 77, zyx, box == 11)
  return cases


def reseg64_cases():
  """The pair and the endpoint result of the reseg_64 process_point run, rebuilt as result files."""
  g = np.load(os.path.join(HERE, 'reseg_64.npz'), allow_pickle=True)
  seg = np.load(os.path.join(HERE, 'flood_fill_64.npz'))['segmentation']
  seg = np.where(seg < 0, 0, seg)[np.newaxis]   # map keys are uint64: -1 (invalid) marks become background
  z, y, x = (int(v) for v in g['point_zyx'])
  radius = tuple(int(v) for v in g['radius_zyx'])
  analysis = tuple(int(v) for v in g['analysis_radius_zyx'])
  cases = []
  for kind in ('pair', 'endpoint'):
    n = int(g[kind + '_n_objects'])
    dels = [g['%s_deletes_%d' % (kind, k)] for k in range(n)]
    hist = [g['%s_history_%d' % (kind, k)] for k in range(n)]
    same = len({d.shape for d in dels}) == 1
    starts = as_object([g['%s_starts_%d' % (kind, k)] for k in range(2)])
    data = write_file(g[kind + '_probs'], np.stack(dels) if same else as_object(dels),
                      np.stack(hist) if same else as_object(hist), starts)
    ida, idb = int(g['id_a']), int(g['id_b']) if kind == 'pair' else 0
    cases.append(dict(name='%d-%d_at_%d_%d_%d.npz' % (ida, idb, x, y, z), kind=kind, file=data, radius=radius,
                      analysis=analysis, voxel=(4, 3, 3), threshold=0.5, tag='reseg64_' + kind))
  return seg, cases


def main():
  import tempfile
  ref = reference_module()
  vol = synthetic_volume()
  seg64, c64 = reseg64_cases()
  volumes = [vol, seg64]
  cases = [(0, c) for c in synthetic_cases(vol)] + [(1, c) for c in c64]
  tmp = tempfile.mkdtemp(prefix='reseg_analysis_golden_')
  out = {'n': len(cases), 'volume_0': vol, 'volume_1': seg64}
  for i, (v, c) in enumerate(cases):
    path = os.path.join(tmp, '%02d' % i, c['name'])
    os.makedirs(os.path.dirname(path))
    with open(path, 'wb') as f:
      f.write(c['file'])
    error, expect = '', b''
    try:
      if c['kind'] == 'pair':
        res = ref.evaluate_pair_resegmentation(path, VolumeStore(volumes[v]), c['radius'], c['analysis'], c['voxel'],
                                               threshold=c['threshold'])
      else:
        res = ref.evaluate_endpoint_resegmentation(path, VolumeStore(volumes[v]), c['radius'], threshold=c['threshold'])
      expect = res.SerializeToString(deterministic=True)
    except (ref.InvalidBaseSegmentatonError, ref.IncompleteResegmentationError) as e:
      error = type(e).__name__
    print('%-22s %-8s %s' % (c['tag'], c['kind'], error or '%d bytes' % len(expect)))
    out.update({
        'tag_%d' % i: c['tag'], 'name_%d' % i: c['name'], 'kind_%d' % i: c['kind'], 'volume_%d_of' % i: v,
        'file_%d' % i: np.frombuffer(c['file'], np.uint8), 'radius_%d' % i: np.array(c['radius']),
        'analysis_%d' % i: np.array(c['analysis']), 'voxel_%d' % i: np.array(c['voxel']),
        'threshold_%d' % i: c['threshold'], 'expect_%d' % i: np.frombuffer(expect, np.uint8), 'error_%d' % i: error})
  np.savez_compressed(OUT, **out)
  print('wrote', OUT)


if __name__ == '__main__':
  main()
