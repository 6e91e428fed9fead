"""PolicyPeaks2d / PolicyFillEmptySpace / PolicyMaxPeaks on the host (ffn/inference/seed.py:202-352): the scipy
path of ffn_b200 and the oracle against the reference's own policies (tests/golden/peak_policies_ref.npz, written by
make_golden_peak_policies.py), and resolution by name as Runner, SequentialPolicies and ReverseCoords do it."""

import functools
import json
import os
import types

import numpy as np
import pytest

from ffn.inference import inference_pb2, runner as runner_mod, seed
from oracle import seed_policies


@pytest.fixture(scope='module')
def ref(golden_dir):
  return np.load(os.path.join(golden_dir, 'peak_policies_ref.npz'))


CASES = ['p2d_default', 'p2d_md3_desc', 'p2d_masked', 'fill', 'max_excl', 'max_rel']


class _Restrictor:
  def __init__(self, mask=None, seed_mask=None):
    self.mask, self.seed_mask = mask, seed_mask


class _HostCanvas:
  """What the host path of a seed policy reads from a canvas (no `_dev`)."""

  def __init__(self, image, segmentation, mask=None, seed_mask=None, margin=(0, 0, 0)):
    self.image, self.segmentation = image, segmentation
    self.restrictor = _Restrictor(mask, seed_mask)
    self.margin, self.shape, self.voxel_size_zyx = np.asarray(margin), image.shape, (1, 1, 1)


def _image(vol):
  return (vol.astype(np.float32) - np.float32(128.0)) / np.float32(33.0)


def _case(ref, case):
  get = lambda k: ref[case + k] if case + k in ref else None   # noqa: E731
  return dict(policy=str(ref[case + '_policy']), kwargs=json.loads(str(ref[case + '_kwargs'])),
              image=_image(ref[case + '_volume']), segmentation=ref[case + '_segmentation'], mask=get('_mask'),
              seed_mask=get('_seed_mask'), margin=ref[case + '_margin'], coords=ref[case + '_coords'])


def _oracle(c, margin):
  if c['policy'] == 'PolicyPeaks2d':
    return seed_policies.policy_peaks_2d(c['image'], mask=c['mask'], margin_zyx=margin, **c['kwargs'])
  if c['policy'] == 'PolicyFillEmptySpace':
    return seed_policies.policy_fill_empty_space(c['segmentation'], margin_zyx=margin)
  return seed_policies.policy_max_peaks(c['image'], c['segmentation'], c['mask'], c['seed_mask'], margin_zyx=margin,
                                        **c['kwargs'])


def test_fixture_covers_every_case(ref):
  assert list(ref['cases']) == CASES
  for case in CASES:
    assert ref[case + '_coords'].shape[0] > 5, case


@pytest.mark.parametrize('case', CASES)
def test_host_policy_equals_reference(ref, case):
  """The scipy path yields exactly the reference's list, order included (Runner's extra kwargs accepted)."""
  c = _case(ref, case)
  cv = _HostCanvas(c['image'], c['segmentation'], c['mask'], c['seed_mask'], c['margin'])
  pol = getattr(seed, c['policy'])(cv, corner=(0, 0, 0), subvol_size=c['image'].shape[::-1], **c['kwargs'])
  got = np.array([tuple(v) for v in pol], dtype=np.int64).reshape(-1, 3)
  np.testing.assert_array_equal(got, c['coords'])


@pytest.mark.parametrize('case', CASES)
def test_oracle_equals_reference(ref, case):
  c = _case(ref, case)
  np.testing.assert_array_equal(_oracle(c, c['margin']), c['coords'])


def test_fixture_shows_what_each_policy_excludes(ref):
  """PolicyPeaks2d proposes seeds in labelled and seed-masked voxels (only the movement mask acts); the
  descending case is reverse-sorted; PolicyMaxPeaks finds peaks of the noise inside its zeroed exclusion."""
  c = _case(ref, 'p2d_masked')
  z, y, x = c['coords'].T
  assert not c['mask'][z, y, x].any()
  assert (c['segmentation'][z, y, x] > 0).any() and c['seed_mask'][z, y, x].any()
  d = [tuple(r) for r in ref['p2d_md3_desc_coords']]
  assert d == sorted(d, reverse=True)
  c = _case(ref, 'fill')
  z, y, x = c['coords'].T
  assert (c['segmentation'][z, y, x] == 0).all() and (c['segmentation'] == -1).any()


def test_no_finite_distance_yields_no_seeds():
  """A slice without edge voxels (PolicyPeaks2d) and a canvas without labelled voxels (PolicyFillEmptySpace) have
  no finite distance: they contribute no seeds, on the host path and in the oracle alike."""
  from ffn_b200.synthetic import voronoi_phantom
  vol = voronoi_phantom((6, 64, 64), seed=4, sigma=(0.5, 1, 1), voxel_size_zyx=(4, 1, 1), cell_volume=6000.0)
  image = _image(vol)
  image[2] = 0.5                                            # a flat slice: no gradient, no edge
  cv = _HostCanvas(image, np.zeros(image.shape, np.int32))
  got = seed.PolicyPeaks2d(cv, min_distance=3, threshold_abs=0).remaining()
  assert got.shape[0] > 10 and 2 not in set(got[:, 0].tolist())
  np.testing.assert_array_equal(got, seed_policies.policy_peaks_2d(image, min_distance=3, threshold_abs=0,
                                                                   margin_zyx=(0, 0, 0)))
  assert seed.PolicyFillEmptySpace(cv).remaining().shape == (0, 3)
  assert seed_policies.policy_fill_empty_space(cv.segmentation).shape == (0, 3)


_PEAKS_REF = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'policy_peaks_ref.npz')
with np.load(_PEAKS_REF) as _r:
  PEAKS_CASES = sorted(k[:-len('_coords')] for k in _r.files if k.endswith('_coords'))


@pytest.mark.parametrize('case', PEAKS_CASES)
def test_host_policy_peaks_equals_reference(case):
  """The scipy path of PolicyPeaks (a canvas without a device) yields exactly the reference's list
  (tests/golden/policy_peaks_ref.npz), order included.  The cases with canvas margins below 3 pin the border
  exclusion of peak_local_max: a peak 1 or 2 voxels from the array border is never a seed."""
  r = np.load(_PEAKS_REF)
  get = lambda k: r[case + k] if case + k in r.files else None   # noqa: E731
  cv = _HostCanvas(_image(r[case + '_volume']), r[case + '_segmentation'], get('_mask'), get('_seed_mask'),
                   r[case + '_margin'])
  cv.voxel_size_zyx = tuple(float(v) for v in r[case + '_voxel'])
  got = np.array([tuple(v) for v in seed.PolicyPeaks(cv)], dtype=np.int64).reshape(-1, 3)
  want = r[case + '_coords']
  assert want.shape[0] >= 5
  np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize('threshold_abs,threshold_rel', [(None, None), (None, 0.3), (0.2, None), (-1.0, 0.6)])
def test_peak_thresholds_follow_peak_local_max(threshold_abs, threshold_rel):
  """threshold_abs=None is the minimum and threshold_rel=None no relative threshold, as in skimage."""
  rng = np.random.RandomState(8)
  values = rng.randn(12, 20, 22).astype(np.float32)
  keys = values + np.random.RandomState(42).rand(*values.shape) * 1e-4
  got = seed._local_peaks(keys, 2, threshold_abs, threshold_rel)   # pylint: disable=protected-access
  np.testing.assert_array_equal(got, seed_policies.peak_local_max_full(keys, 2, threshold_abs, threshold_rel))
  assert got.shape[0] > 3


def test_policies_resolve_by_name_in_runner_sequential_and_reverse(ref):
  c = _case(ref, 'fill')                                   # a mostly labelled canvas, so that there are gaps to fill
  c['mask'] = np.zeros(c['image'].shape, dtype=bool)
  c['mask'][:, :, :8] = True
  kw = {'min_distance': 3, 'threshold_abs': 0.5}
  cv = _HostCanvas(c['image'], c['segmentation'], c['mask'], None, c['margin'])
  for name in ('PolicyPeaks2d', 'PolicyFillEmptySpace', 'PolicyMaxPeaks'):
    req = inference_pb2.InferenceRequest(seed_policy=name, seed_policy_args=json.dumps(kw) if name == 'PolicyPeaks2d'
                                         else '')
    factory = runner_mod.Runner.get_seed_policy(types.SimpleNamespace(request=req), (0, 0, 0), (52, 48, 28))
    assert isinstance(factory, functools.partial) and factory.func is getattr(seed, name)
    pol = factory(cv)
    assert isinstance(pol, getattr(seed, name)) and pol.remaining().shape[0] > 0
  p2d = seed_policies.policy_peaks_2d(c['image'], mask=c['mask'], margin_zyx=c['margin'], **kw)
  fill = seed_policies.policy_fill_empty_space(c['segmentation'], margin_zyx=c['margin'])
  maxp = seed_policies.policy_max_peaks(c['image'], c['segmentation'], c['mask'], margin_zyx=c['margin'])
  np.testing.assert_array_equal(fill, c['coords'])
  seq = seed.SequentialPolicies(cv, [['PolicyPeaks2d', kw], ['PolicyFillEmptySpace', {}], ['PolicyMaxPeaks', {}]])
  np.testing.assert_array_equal(seq.remaining(), np.concatenate([p2d, fill, maxp]))
  rev = seed.ReverseCoords(cv, 'PolicyPeaks2d', **kw)
  np.testing.assert_array_equal(rev.remaining(), p2d[::-1])
  rev = seed.ReverseCoords(cv, 'PolicyMaxPeaks', min_distance=3)
  np.testing.assert_array_equal(rev.remaining(), maxp[::-1])
