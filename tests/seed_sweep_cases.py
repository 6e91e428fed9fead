"""The seed-policy sweep: canvases, masks and parameters at which the device seed policies (seedk:: kernels behind
ffn_canvas_seed_peaks / ffn_canvas_seed_policy) are compared with the scipy oracle (test_gpu_seed_sweep.py), and at
which plausible kernel defects are shown to change the oracle's answer (test_seed_sweep_oracle.py).

Every case is built deterministically from its name.  `kind` is 'peaks' (PolicyPeaks), or one of the
ffn_canvas_seed_policy kinds 'peaks_2d', 'fill_empty', 'max_peaks'.  `min_peaks` is the least number of RAW peaks
(before any canvas-margin filter) the oracle must find, and `exact_zero` marks the cases whose definition is "no
peaks at all"."""

import numpy as np

from ffn_b200.synthetic import voronoi_phantom


def _u8(shape, seed, cell_volume=3000.0, sigma=(1.0, 1.0, 1.0)):
  return voronoi_phantom(shape, seed=seed, sigma=sigma, cell_volume=cell_volume)


def _f32(vol, mean=128.0, std=33.0):
  return (vol.astype(np.float32) - np.float32(mean)) / np.float32(std)


def _blocks(shape, seed, block=4, levels=5):
  """Float32 image of constant blocks (exact ties, plateaus) with a few levels."""
  rng = np.random.RandomState(seed)
  small = rng.randint(0, levels, size=tuple(-(-s // block) for s in shape)).astype(np.float32) * np.float32(0.75)
  return np.ascontiguousarray(np.kron(small, np.ones((block,) * 3, np.float32))[tuple(slice(0, s) for s in shape)])


def _sparse_edges(shape, seed):
  """u8 canvas of constant 128 with two flat membrane-like slabs near both x ends and a few bright spots beside
  them: an edge-free gap of hundreds of voxels along x, whose mid-plane is a plateau of equal distances."""
  rng = np.random.RandomState(seed)
  vol = np.full(shape, 128, np.uint8)
  for x0 in (6, shape[2] - 7):
    vol[:, :, x0 - 1:x0 + 2] = 40
  for _ in range(6):
    cz, cy = rng.randint(2, shape[0] - 2), rng.randint(4, shape[1] - 4)
    cx = rng.randint(20, 40) if rng.rand() < 0.5 else shape[2] - rng.randint(20, 40)
    vol[max(cz - 1, 0):cz + 2, cy - 2:cy + 3, cx - 2:cx + 3] = 230
  return vol


# (name, kind, builder, params); params default: voxel (1, 1, 1), min_distance / thresholds of the policy defaults.
def _case_specs():
  specs = []

  def add(name, kind, **kw):
    specs.append(dict(name=name, kind=kind, **kw))

  # ---- PolicyPeaks: Sobel + gaussian + EDT (voxel size) + 7^3 peaks with the 3-voxel border exclusion ----
  add('peaks_z1', 'peaks', shape=(1, 40, 52), image='u8', seed=31, exact_zero=True)
  add('peaks_z2', 'peaks', shape=(2, 37, 41), image='u8', seed=32, exact_zero=True)
  add('peaks_x3', 'peaks', shape=(20, 37, 3), image='f32q', seed=33, exact_zero=True)
  add('peaks_small', 'peaks', shape=(9, 20, 29), image='f32', seed=34, cell=1500.0, min=1)
  add('peaks_prime_123', 'peaks', shape=(17, 97, 101), image='u8', seed=35, mean=127.5, std=31.7, voxel=(1, 2, 3))
  add('peaks_iso_masks', 'peaks', shape=(32, 72, 80), image='u8', seed=36, masks=True)
  add('peaks_aniso_211', 'peaks', shape=(24, 61, 67), image='u8', seed=37, voxel=(2, 1, 1), cell=2000.0)
  add('peaks_f32q_30_8_8', 'peaks', shape=(24, 60, 64), image='f32q', seed=38, voxel=(30, 8, 8))
  add('peaks_f32blocks', 'peaks', shape=(20, 36, 44), image='blocks', seed=39, masks=True)
  add('peaks_grid_stride', 'peaks', shape=(40, 130, 600), image='u8', seed=40, voxel=(2, 1, 1), cell=6000.0)
  add('peaks_em_40_16_16', 'peaks', shape=(24, 96, 700), image='sparse', seed=41, voxel=(40, 16, 16))
  add('peaks_em_9_7_15', 'peaks', shape=(24, 96, 700), image='sparse', seed=41, voxel=(9, 7, 15))
  add('peaks_all_masked', 'peaks', shape=(12, 30, 34), image='u8', seed=42, all_blocked=True, exact_zero=True)

  # ---- PolicyPeaks2d: per-slice 2-D Sobel + gaussian + EDT, peaks with the in-plane border ----
  add('p2d_z1_md3', 'peaks_2d', shape=(1, 40, 52), image='u8', seed=51, md=3, thr=0.0)
  add('p2d_z2_md1_none', 'peaks_2d', shape=(2, 37, 41), image='u8', seed=52, md=1, thr=None)
  add('p2d_x3_md1', 'peaks_2d', shape=(9, 40, 3), image='f32q', seed=53, md=1, thr=0.0)
  add('p2d_small_md0_none', 'peaks_2d', shape=(7, 20, 29), image='u8', seed=54, md=0, thr=None, cell=400.0)
  add('p2d_small_md0_zero', 'peaks_2d', shape=(7, 20, 29), image='u8', seed=54, md=0, thr=0.0, cell=400.0)
  add('p2d_prime_md3_masked', 'peaks_2d', shape=(17, 97, 101), image='u8', seed=55, md=3, thr=2.5, masks=True,
      mean=127.5, std=31.7)
  add('p2d_md7_flat_slice', 'peaks_2d', shape=(6, 64, 70), image='f32', seed=56, md=7, thr=0.0, flat_slice=2)
  add('p2d_md7_default', 'peaks_2d', shape=(8, 90, 96), image='u8', seed=57, md=7, thr=2.5)
  add('p2d_md_over_half_y', 'peaks_2d', shape=(5, 30, 64), image='u8', seed=58, md=16, thr=0.0, exact_zero=True)
  add('p2d_grid_stride_none', 'peaks_2d', shape=(40, 130, 600), image='u8', seed=40, md=3, thr=None, cell=6000.0)

  # ---- PolicyFillEmptySpace: EDT of the unlabelled voxels, peaks at min_distance 2 above 0.5 ----
  add('fill_single_label', 'fill_empty', shape=(20, 30, 40), seg='single', exact_zero=True)
  add('fill_almost_full', 'fill_empty', shape=(16, 24, 28), seg='almost_full')
  add('fill_markers_only', 'fill_empty', shape=(18, 40, 44), seg='markers')
  add('fill_cells', 'fill_empty', shape=(17, 97, 101), seg='cells', seed=59)

  # ---- PolicyMaxPeaks: image intensity with the excluded voxels zeroed ----
  add('max_md0_none_none', 'max_peaks', shape=(2, 37, 41), image='f32fine', seed=61, md=0, thr=None, rel=None)
  add('max_md1_x3', 'max_peaks', shape=(12, 40, 3), image='f32fine', seed=62, md=1, thr=0.0, rel=None)
  add('max_md3_masks', 'max_peaks', shape=(17, 97, 101), image='u8', seed=63, md=3, thr=0.3, rel=None, masks=True,
      mean=127.5, std=31.7)
  add('max_md9_grid_stride', 'max_peaks', shape=(40, 130, 600), image='u8', seed=40, md=9, thr=None, rel=0.0,
      cell=6000.0)
  add('max_md3_fine', 'max_peaks', shape=(16, 40, 44), image='f32fine', seed=64, md=3, thr=0.0, rel=0.0)
  add('max_md1_blocks', 'max_peaks', shape=(20, 36, 44), image='blocks', seed=65, md=1, thr=None, rel=0.4, masks=True)
  add('max_md0_thr', 'max_peaks', shape=(7, 20, 29), image='f32q', seed=66, md=0, thr=0.3, rel=0.4, cell=400.0)
  return specs


SPECS = {s['name']: s for s in _case_specs()}
NAMES = list(SPECS)


def min_peaks(name):
  """The least number of raw peaks a case must have (0 for the cases defined to have none)."""
  s = SPECS[name]
  return 0 if s.get('exact_zero') else s.get('min', 3)


def build(name):
  """The case's arrays and parameters: image (u8 or float32), mean / std (u8 only), image_f32 (what the policies
  see), voxel, segmentation, mask, seed_mask (or None), min_distance, threshold_abs, threshold_rel."""
  s = dict(SPECS[name])
  shape = tuple(s['shape'])
  seed = s.get('seed', 0)
  mean, std = s.get('mean', 128.0), s.get('std', 33.0)
  kind_img = s.get('image', 'u8')
  cell = s.get('cell', 3000.0)
  if kind_img == 'u8':
    image = _u8(shape, seed, cell)
  elif kind_img == 'f32':
    image = _f32(_u8(shape, seed, cell))
  elif kind_img == 'f32q':
    image = np.round(_f32(_u8(shape, seed, cell)) * np.float32(2)) / np.float32(2)     # quantised: exact ties
  elif kind_img == 'f32fine':
    rng = np.random.RandomState(seed)
    image = (np.float32(1.0) + np.float32(2e-5) * rng.randn(*shape).astype(np.float32)).astype(np.float32)
  elif kind_img == 'blocks':
    image = _blocks(shape, seed)
  else:
    image = _sparse_edges(shape, seed)
  if 'flat_slice' in s:
    image[s['flat_slice']] = image.dtype.type(100 if image.dtype == np.uint8 else 0.5)
  image_f32 = _f32(image, mean, std) if image.dtype == np.uint8 else image.astype(np.float32)

  rng = np.random.RandomState(1000 + seed)
  seg = np.zeros(shape, np.int32)
  mask = seed_mask = None
  if s.get('masks'):
    mask = np.zeros(shape, bool)
    mask[:, :max(shape[1] // 6, 1), :] = True
    seed_mask = rng.rand(*shape) > 0.97
    seed_mask[:, shape[1] // 2:shape[1] // 2 + 5, shape[2] // 3:shape[2] // 3 + 7] = True
    seg[shape[0] // 4:shape[0] // 2 + 1, shape[1] // 3:2 * shape[1] // 3, shape[2] // 2:] = 5
    k = max(np.prod(shape) // 400, 4)
    seg[rng.randint(0, shape[0], k), rng.randint(0, shape[1], k), rng.randint(0, shape[2], k)] = -1
  if s.get('all_blocked'):
    mask = np.zeros(shape, bool)
    mask[:, :shape[1] // 2] = True
    seed_mask = ~mask                                  # every voxel is either masked or seed-masked
  which = s.get('seg')
  if which == 'single':
    seg[shape[0] // 3, shape[1] // 2, shape[2] // 4] = 3
  elif which == 'almost_full':
    seg[...] = 1
    for z, y, x in ((5, 6, 7), (8, 12, 20), (10, 3, 14), (12, 18, 9), (6, 20, 24)):
      seg[z, y, x] = 0
  elif which == 'markers':
    k = 400
    seg[rng.randint(0, shape[0], k), rng.randint(0, shape[1], k), rng.randint(0, shape[2], k)] = -1
  elif which == 'cells':
    _, cells = voronoi_phantom(shape, seed=seed, cell_volume=4000.0, return_cells=True)
    ids = np.unique(cells[cells > 0])
    for k, cid in enumerate(ids[rng.rand(ids.size) < 0.5]):
      seg[cells == cid] = k + 1
    seg[rng.rand(*shape) > 0.998] = -1
  if s['kind'] == 'fill_empty':                         # the image does not enter PolicyFillEmptySpace
    image = np.full(shape, 128, np.uint8)
    image_f32 = _f32(image, mean, std)
  return dict(name=name, kind=s['kind'], image=image, mean=mean, std=std, image_f32=image_f32,
              voxel=tuple(float(v) for v in s.get('voxel', (1, 1, 1))), segmentation=seg, mask=mask,
              seed_mask=seed_mask, min_distance=s.get('md'), threshold_abs=s.get('thr', 0.0),
              threshold_rel=s.get('rel', 0.0), exact_zero=bool(s.get('exact_zero')))


def noise(case):
  """The tie-break noise exactly as the policy draws it: RandomState(42).rand of the canvas, or of the (Y, X) plane
  for PolicyPeaks2d."""
  shape = case['image'].shape
  return np.random.RandomState(seed=42).rand(*(shape[1:] if case['kind'] == 'peaks_2d' else shape))


def oracle(case):
  """The oracle's RAW peak list (no canvas margin), lexicographically sorted."""
  from oracle import seed_peaks, seed_policies
  k = case['kind']
  if k == 'peaks':
    out = seed_peaks.policy_peaks(case['image_f32'], case['voxel'], segmentation=case['segmentation'],
                                  mask=case['mask'], seed_mask=case['seed_mask'])
  elif k == 'peaks_2d':
    out = seed_policies.policy_peaks_2d(case['image_f32'], mask=case['mask'], min_distance=case['min_distance'],
                                        threshold_abs=case['threshold_abs'])
  elif k == 'fill_empty':
    out = seed_policies.policy_fill_empty_space(case['segmentation'])
  else:
    out = seed_policies.policy_max_peaks(case['image_f32'], case['segmentation'], case['mask'], case['seed_mask'],
                                         min_distance=case['min_distance'], threshold_abs=case['threshold_abs'],
                                         threshold_rel=case['threshold_rel'])
  return lexsorted(out)


def lexsorted(coords):
  c = np.asarray(coords, dtype=np.int64).reshape(-1, 3)
  return c[np.lexsort((c[:, 2], c[:, 1], c[:, 0]))]
