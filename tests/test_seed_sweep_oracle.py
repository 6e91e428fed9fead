"""The seed-policy sweep (seed_sweep_cases.py, run on the device by test_gpu_seed_sweep.py) is sensitive to the kernel
defects that are easy to make in the seedk:: kernels: each defect, applied to a restatement of the oracle, changes at
least one case's raw peak list.

`_policy` restates oracle/seed_peaks.py and oracle/seed_policies.py from the same stages the kernels implement
(Sobel + gaussian edge map, exact EDT, (dt, noise) keys, box maximum, thresholds, border exclusion); without a
defect it must equal the oracle on every case, so a defect it exposes is one the device sweep would expose."""

import numpy as np
import pytest
from scipy import ndimage

import seed_sweep_cases as sc

DEFECTS = ['nearest_boundary', 'voxel_axes_swapped', 'lexicographic_keys', 'no_border', 'canvas_wide_min_2d']


def _edges(image, nearest):
  """oracle.seed_peaks.edge_map, optionally with 'nearest' instead of 'reflect' at the boundary."""
  mode = 'nearest' if nearest else 'reflect'
  grad = ndimage.generic_gradient_magnitude(np.asarray(image, np.float32), ndimage.sobel, mode=mode)
  thresh = np.zeros(grad.shape, np.float32)
  ndimage.gaussian_filter(grad, 49.0 / 6.0, output=thresh, mode=mode)
  return grad > thresh


def _edt(foreground, sampling, f32_squared):
  """Exact EDT (float32 result); optionally with the squared distance rounded to float32 before the square root."""
  if not f32_squared:
    return ndimage.distance_transform_edt(foreground, sampling=sampling).astype(np.float32)
  idx = ndimage.distance_transform_edt(foreground, sampling=sampling, return_distances=False, return_indices=True)
  grid = np.indices(foreground.shape)
  d2 = sum(((idx[a] - grid[a]) * float(sampling[a])) ** 2 for a in range(foreground.ndim))
  return np.sqrt(d2.astype(np.float32))


def _peaks(values, noise, min_distance, threshold, lexicographic, border):
  """Peaks of (values, noise): key == box maximum, key > threshold, at least `border` voxels from the border.  The
  key is values + noise * 1e-4 in float64, or (values, noise) compared lexicographically."""
  values = np.asarray(values, np.float32)
  keys = values.astype(np.float64) + noise * 1e-4
  if lexicographic:          # dense rank of the value + noise in [0, 1): float64 order == lexicographic order
    finite = np.isfinite(values)
    rank = np.full(values.shape, -np.inf)
    rank[finite] = np.unique(values[finite], return_inverse=True)[1].reshape(-1).astype(np.float64) + 2.0
    order = np.where(finite, rank + noise, -np.inf)
  else:
    order = keys
  ok = np.isfinite(keys)
  keep = ok & (order == ndimage.maximum_filter(order, size=2 * min_distance + 1, mode='nearest')) & (keys > threshold)
  if border:
    inner = np.zeros(values.shape, bool)
    inner[tuple(slice(border, s - border) for s in values.shape)] = True
    keep &= inner
  return np.argwhere(keep)


def _threshold(keys, threshold_abs, threshold_rel):
  finite = keys[np.isfinite(keys)]
  if not finite.size:
    return np.inf
  thr = float(finite.min()) if threshold_abs is None else float(threshold_abs)
  if threshold_rel is not None:
    thr = max(thr, float(threshold_rel) * float(finite.max()))
  return thr


def _policy(c, defect=None):
  """The case's raw peak list, with at most one defect."""
  kind, nz = c['kind'], sc.noise(c)
  border = lambda md: 0 if defect == 'no_border' else md   # noqa: E731
  lex = defect == 'lexicographic_keys'
  if kind == 'peaks':
    edges = _edges(c['image_f32'], defect == 'nearest_boundary')
    excl = c['segmentation'] > 0
    for m in (c['mask'], c['seed_mask']):
      if m is not None:
        excl |= m
        edges |= m
    if edges.all():
      return np.zeros((0, 3), np.int64)
    voxel = c['voxel'][::-1] if defect == 'voxel_axes_swapped' else c['voxel']
    dt = _edt(~edges, voxel, defect == 'f32_squared_distance')
    dt[excl | ~np.isfinite(dt)] = -1
    return sc.lexsorted(_peaks(dt, nz, 3, 0.0, lex, border(3)))
  if kind == 'peaks_2d':
    md = c['min_distance']
    dts = []
    for z in range(c['image_f32'].shape[0]):
      edges = _edges(c['image_f32'][z], defect == 'nearest_boundary')
      if c['mask'] is not None:
        edges |= c['mask'][z]
      dts.append(_edt(~edges, (1.0, 1.0), defect == 'f32_squared_distance') if edges.any()
                 else np.full(edges.shape, np.inf, np.float32))
    canvas_keys = np.stack(dts).astype(np.float64) + nz[None] * 1e-4
    rows = []
    for z, dt in enumerate(dts):
      keys = canvas_keys if defect == 'canvas_wide_min_2d' else canvas_keys[z]
      thr = _threshold(keys, c['threshold_abs'], 0)
      rows += [(z, y, x) for y, x in _peaks(dt, nz, md, thr, lex, border(md))]
    return sc.lexsorted(rows)
  if kind == 'fill_empty':
    seg = c['segmentation']
    if (seg == 0).all():
      return np.zeros((0, 3), np.int64)
    dt = _edt(seg == 0, (1.0, 1.0, 1.0), defect == 'f32_squared_distance')
    return sc.lexsorted(_peaks(dt, nz, 2, 0.5, lex, border(2)))
  img = np.array(c['image_f32'], np.float32)
  excl = c['segmentation'] > 0
  for m in (c['mask'], c['seed_mask']):
    if m is not None:
      excl |= m
  img[excl] = 0
  md = c['min_distance']
  thr = _threshold(img.astype(np.float64) + nz * 1e-4, c['threshold_abs'], c['threshold_rel'])
  return sc.lexsorted(_peaks(img, nz, md, thr, lex, border(md)))


@pytest.fixture(scope='module')
def cases():
  return {name: sc.build(name) for name in sc.NAMES}


@pytest.fixture(scope='module')
def oracle_lists(cases):
  return {name: sc.oracle(c) for name, c in cases.items()}


def test_every_case_has_peaks_unless_none_is_the_definition(oracle_lists):
  """No case can pass with two empty lists by accident: each finds peaks, or is defined to find none."""
  for name, got in oracle_lists.items():
    spec = sc.SPECS[name]
    if spec.get('exact_zero'):
      assert got.shape[0] == 0, name
    else:
      assert got.shape[0] >= sc.min_peaks(name), (name, got.shape[0])


def test_restatement_equals_the_oracle(cases, oracle_lists):
  for name, c in cases.items():
    np.testing.assert_array_equal(_policy(c), oracle_lists[name], err_msg=name)


@pytest.mark.parametrize('defect', DEFECTS)
def test_sweep_detects_defect(cases, oracle_lists, defect):
  changed = [name for name, c in cases.items() if not np.array_equal(_policy(c, defect), oracle_lists[name])]
  print('%s changes %d of %d cases: %s' % (defect, len(changed), len(cases), ', '.join(changed)))
  assert changed, defect


def test_float32_squared_distances_change_no_case(cases, oracle_lists):
  """The EDT kernels carry squared distances in float32 (seedk::edt_x / edt_line).  Rounding them to float32 before
  the square root changes no raw list of the sweep, including the peaks_em_* cases whose squared distances exceed
  2^24, where float32 stops holding every integer: competing distances differ by far more than that rounding, and
  exactly tied distances round alike.  So the float32 squared distances stay; this test tells if a case ever proves
  otherwise."""
  for name, c in cases.items():
    if c['kind'] in ('peaks', 'fill_empty'):
      np.testing.assert_array_equal(_policy(c, 'f32_squared_distance'), oracle_lists[name], err_msg=name)
  for name in ('peaks_em_40_16_16', 'peaks_em_9_7_15'):
    c = cases[name]
    edges = _edges(c['image_f32'], False)
    assert ndimage.distance_transform_edt(~edges, sampling=c['voxel']).max() ** 2 > 2.0 ** 24, name
