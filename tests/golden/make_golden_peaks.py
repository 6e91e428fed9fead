"""PolicyPeaks fixture: the REAL reference `ffn.inference.seed.PolicyPeaks` (ffn/inference/seed.py:36-199: `__next__`
border filter, `get_exclusion_mask`, `_find_peaks`, `init_coords`) iterated to exhaustion on small volumes.

    PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION=python python tests/golden/make_golden_peaks.py

The reference module runs unmodified.  Its two UN-VENDORED third-party calls (setup.py:43,47, absent from
/root/reference and from this image) are injected with their published definitions, independently of oracle/ and of
the product:
  * `edt.edt(binary, anisotropy)`  -> exact Euclidean distance transform in physical units (scipy's exact EDT here;
    tests/test_oracle_golden.py pins that to the O(n^2) definition);
  * `skimage.feature.peak_local_max(image, min_distance, threshold_abs, threshold_rel)` -> documented semantics: a
    voxel is a peak iff it equals the maximum over its (2 min_distance + 1)^3 neighbourhood and exceeds the
    threshold; peaks within min_distance of the border are dropped; best first.
So this pins everything the reference's OWN code does around them — Sobel magnitude, adaptive gaussian threshold
(sigma 49/6, reflect), masks counted as edges, the all-edges early return, the exclusion mask (labels, mask, seed_mask),
-1 / non-finite handling, the RandomState(42) tie-break noise, the lexicographic re-sort and the border filter of
`__next__` — and leaves exactly those two definitions unpinned.  Output: policy_peaks_ref.npz (cases iso / aniso /
masked, and the same three volumes with canvas margins below 3, where the border exclusion of peak_local_max alone
decides which peaks near the array border survive).
"""
import os
import sys
import types

import numpy as np
from scipy import ndimage

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402


def edt_definition(binary, anisotropy=(1.0, 1.0, 1.0), **kwargs):
  del kwargs
  return ndimage.distance_transform_edt(np.asarray(binary) != 0, sampling=tuple(float(a) for a in anisotropy))


def peak_local_max_definition(image, min_distance=1, threshold_abs=None, threshold_rel=None, **kwargs):
  del kwargs
  size = 2 * min_distance + 1
  thr = -np.inf
  if threshold_abs is not None:
    thr = max(thr, threshold_abs)
  if threshold_rel is not None:
    thr = max(thr, threshold_rel * image.max())
  peak = (image == ndimage.maximum_filter(image, size=size, mode='nearest')) & (image > thr)
  inner = np.zeros(image.shape, dtype=bool)
  inner[tuple(slice(min_distance, s - min_distance) for s in image.shape)] = True
  idx = np.argwhere(peak & inner)
  order = np.argsort(-image[tuple(idx.T)], kind='stable')
  return idx[order]


def main():
  os.environ.setdefault('PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION', 'python')
  mg.install_stubs()
  sys.path.insert(0, mg.REF)
  from ffn.inference import seed as ref_seed
  from ffn_b200.synthetic import voronoi_phantom

  ref_seed.edt = types.SimpleNamespace(edt=edt_definition)
  ref_seed.skimage = types.SimpleNamespace(feature=types.SimpleNamespace(peak_local_max=peak_local_max_definition))

  class Restrictor:
    def __init__(self, mask=None, seed_mask=None):
      self.mask, self.seed_mask = mask, seed_mask

  class FakeCanvas:
    def __init__(self, image, voxel, restrictor, segmentation, margin):
      self.image = image
      self.voxel_size_zyx = voxel
      self.restrictor = restrictor
      self.segmentation = segmentation
      self.shape = image.shape
      self.margin = np.asarray(margin)

  out = {}
  cases = [
      ('iso', (44, 52, 60), 3, (1.0, 1.0, 1.0), (1.0, 1.0, 1.0), (6, 6, 6), False),
      ('aniso', (28, 56, 60), 4, (0.5, 1.0, 1.0), (2.0, 1.0, 1.0), (4, 6, 6), False),
      ('masked', (44, 52, 60), 5, (1.0, 1.0, 1.0), (1.0, 1.0, 1.0), (4, 4, 4), True),
      # canvas margins below min_distance = 3: only peak_local_max's exclude_border removes the border peaks
      ('iso_m1', (44, 52, 60), 3, (1.0, 1.0, 1.0), (1.0, 1.0, 1.0), (1, 1, 1), False),
      ('aniso_m2', (28, 56, 60), 4, (0.5, 1.0, 1.0), (2.0, 1.0, 1.0), (2, 1, 2), False),
      ('masked_m0', (44, 52, 60), 5, (1.0, 1.0, 1.0), (1.0, 1.0, 1.0), (0, 2, 1), True),
  ]
  for name, shape, seed, sigma, voxel, margin, masked in cases:
    vol = voronoi_phantom(shape, seed=seed, sigma=sigma, voxel_size_zyx=voxel, cell_volume=9000.0)
    image = (vol.astype(np.float32) - np.float32(128.0)) / np.float32(33.0)
    segmentation = np.zeros(shape, dtype=np.int32)
    mask = seed_mask = None
    if masked:
      rng = np.random.RandomState(17)
      mask = np.zeros(shape, dtype=bool)
      mask[:, :14, :] = True                                   # a slab the FoV may not enter
      seed_mask = np.zeros(shape, dtype=bool)
      seed_mask[20:30, 30:44, 20:40] = True                    # a box that may not be seeded
      segmentation[8:20, 20:40, 40:56] = 7                     # an existing object
      segmentation[rng.randint(0, shape[0], 40), rng.randint(0, shape[1], 40), rng.randint(0, shape[2], 40)] = -1
    canvas = FakeCanvas(image, voxel, Restrictor(mask, seed_mask), segmentation, margin)
    policy = ref_seed.PolicyPeaks(canvas)
    coords = np.array([tuple(int(v) for v in c) for c in policy], dtype=np.int64).reshape(-1, 3)
    print(name, shape, 'voxel', voxel, 'margin', margin, '->', coords.shape[0], 'seeds; first', coords[:2].tolist())
    out[name + '_volume'] = vol
    out[name + '_voxel'] = np.asarray(voxel)
    out[name + '_margin'] = np.asarray(margin)
    out[name + '_coords'] = coords
    out[name + '_segmentation'] = segmentation
    if masked:
      out[name + '_mask'] = mask
      out[name + '_seed_mask'] = seed_mask
  # the all-edges early return (seed.py:176-177): everything masked -> no seeds
  shape = (20, 24, 28)
  canvas = FakeCanvas(np.zeros(shape, np.float32), (1, 1, 1), Restrictor(np.ones(shape, bool), None), np.zeros(shape, np.int32),
                      (2, 2, 2))
  assert list(ref_seed.PolicyPeaks(canvas)) == []
  np.savez_compressed(os.path.join(HERE, 'policy_peaks_ref.npz'), **out)
  print('wrote policy_peaks_ref.npz')


if __name__ == '__main__':
  main()
