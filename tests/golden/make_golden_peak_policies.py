"""PolicyPeaks2d / PolicyFillEmptySpace / PolicyMaxPeaks fixture: the REAL reference policies
(ffn/inference/seed.py:202-352, with `_find_peaks` :133-139 and the border filter of `__next__` :81-88) iterated to
exhaustion on small Voronoi phantoms.

    PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION=python python tests/golden/make_golden_peak_policies.py

The reference module runs unmodified.  Its two un-vendored third-party calls are injected with the same published
definitions as make_golden_peaks.py (`edt_definition`, `peak_local_max_definition`, imported from there), so this pins
everything the reference's own code does around them: the 2-D per-slice Sobel / gaussian / threshold, the movement
mask as edges, the 2-D tie-break noise plane, the EDT input of the segmentation, the exclusion mask set to 0, the
thresholds and min_distance forwarded to peak_local_max, the lexicographic (or reversed) sort and the border filter.

Every case keeps at least one edge voxel per z-slice (PolicyPeaks2d) and one labelled voxel (PolicyFillEmptySpace):
with no finite distance at all the result depends on the un-vendored `edt` package and is not pinned here.

Output: peak_policies_ref.npz, per case `<case>_coords` plus the inputs (`_volume`, `_segmentation`, `_mask`,
`_seed_mask`, `_margin`).
"""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402
from make_golden_peaks import edt_definition, peak_local_max_definition  # noqa: E402

# (name, policy, kwargs, shape, phantom seed, phantom sigma, phantom voxel size, margin, extras)
CASES = [
    ('p2d_default', 'PolicyPeaks2d', {}, (10, 96, 104), 11, (0.5, 1.0, 1.0), (4.0, 1.0, 1.0), (2, 5, 5), ()),
    ('p2d_md3_desc', 'PolicyPeaks2d', {'min_distance': 3, 'threshold_abs': 0, 'sort_cmp': 'descending'},
     (8, 60, 68), 12, (0.5, 1.0, 1.0), (4.0, 1.0, 1.0), (1, 2, 2), ()),
    ('p2d_masked', 'PolicyPeaks2d', {'min_distance': 4, 'threshold_abs': 1.0}, (8, 72, 80), 13, (0.5, 1.0, 1.0),
     (4.0, 1.0, 1.0), (1, 3, 3), ('mask', 'seed_mask', 'labels')),
    ('fill', 'PolicyFillEmptySpace', {}, (28, 48, 52), 14, (1.0, 1.0, 1.0), (1.0, 1.0, 1.0), (1, 1, 1),
     ('blobs',)),
    ('max_excl', 'PolicyMaxPeaks', {}, (24, 40, 44), 15, (1.0, 1.0, 1.0), (1.0, 1.0, 1.0), (1, 2, 2),
     ('mask', 'seed_mask', 'labels')),
    ('max_rel', 'PolicyMaxPeaks', {'threshold_rel': 0.5, 'min_distance': 4}, (24, 40, 44), 16, (1.0, 1.0, 1.0),
     (1.0, 1.0, 1.0), (2, 2, 2), ()),
]


def edt_nd(binary, anisotropy=None, **kwargs):
  """edt.edt's default anisotropy is unit spacing for any rank (PolicyPeaks2d calls it on 2-D slices)."""
  if anisotropy is None:
    anisotropy = (1.0,) * np.ndim(binary)
  return edt_definition(binary, anisotropy=anisotropy, **kwargs)


def case_inputs(shape, seed, sigma, voxel, extras):
  from ffn_b200.synthetic import voronoi_phantom
  vol, cells = voronoi_phantom(shape, seed=seed, sigma=sigma, voxel_size_zyx=voxel, cell_volume=6000.0,
                               return_cells=True)
  rng = np.random.RandomState(seed + 100)
  segmentation = np.zeros(shape, dtype=np.int32)
  mask = seed_mask = None
  z, y, x = shape
  if 'mask' in extras:
    mask = np.zeros(shape, dtype=bool)
    mask[:, :, :x // 5] = True                                  # a slab the FoV may not enter
  if 'seed_mask' in extras:
    seed_mask = np.zeros(shape, dtype=bool)
    seed_mask[:, y // 2:y // 2 + 12, x // 2:x // 2 + 14] = True   # a box that may not be seeded
  if 'labels' in extras:
    segmentation[:, 4:y // 3, x // 2:] = 9                      # an existing object
  if 'blobs' in extras:
    ids = np.unique(cells[cells > 0])
    ids = ids[rng.rand(ids.size) < 0.6]
    for k, cid in enumerate(ids):                               # most cells already segmented
      segmentation[cells == cid] = k + 1
  if 'blobs' in extras or 'labels' in extras:
    n = 30                                                      # -1 markers (rejected seeds)
    segmentation[rng.randint(0, z, n), rng.randint(0, y, n), rng.randint(0, x, n)] = -1
  return vol, segmentation, mask, seed_mask


def main():
  os.environ.setdefault('PROTOCOL_BUFFERS_PYTHON_IMPLEMENTATION', 'python')
  mg.install_stubs()
  sys.path.insert(0, mg.REF)
  from ffn.inference import seed as ref_seed

  ref_seed.edt = types.SimpleNamespace(edt=edt_nd)
  ref_seed.skimage = types.SimpleNamespace(feature=types.SimpleNamespace(peak_local_max=peak_local_max_definition))

  class Restrictor:
    def __init__(self, mask=None, seed_mask=None):
      self.mask, self.seed_mask = mask, seed_mask

  class FakeCanvas:
    def __init__(self, image, restrictor, segmentation, margin):
      self.image = image
      self.voxel_size_zyx = (1.0, 1.0, 1.0)
      self.restrictor = restrictor
      self.segmentation = segmentation
      self.shape = image.shape
      self.margin = np.asarray(margin)

  out = {}
  for name, policy, kwargs, shape, seed, sigma, voxel, margin, extras in CASES:
    vol, segmentation, mask, seed_mask = case_inputs(shape, seed, sigma, voxel, extras)
    image = (vol.astype(np.float32) - np.float32(128.0)) / np.float32(33.0)
    canvas = FakeCanvas(image, Restrictor(mask, seed_mask), segmentation, margin)
    pol = getattr(ref_seed, policy)(canvas, corner=(0, 0, 0), subvol_size=shape[::-1], **kwargs)
    coords = np.array([tuple(int(v) for v in c) for c in pol], dtype=np.int64).reshape(-1, 3)
    if policy == 'PolicyPeaks2d':
      assert len(np.unique(coords[:, 0])) > 1, name
    print(name, policy, kwargs, shape, 'margin', margin, '->', coords.shape[0], 'seeds; first', coords[:2].tolist())
    assert coords.shape[0] > 5, name
    out[name + '_policy'] = np.asarray(policy)
    out[name + '_kwargs'] = np.asarray(json.dumps(kwargs))
    out[name + '_volume'] = vol
    out[name + '_margin'] = np.asarray(margin)
    out[name + '_segmentation'] = segmentation
    out[name + '_coords'] = coords
    if mask is not None:
      out[name + '_mask'] = mask
    if seed_mask is not None:
      out[name + '_seed_mask'] = seed_mask
  out['cases'] = np.asarray([c[0] for c in CASES])
  np.savez_compressed(os.path.join(HERE, 'peak_policies_ref.npz'), **out)
  print('wrote peak_policies_ref.npz')


if __name__ == '__main__':
  main()
