"""find_decision_points on the device (ffn_decision_points): against the reference's own function
(tests/golden/decision_points_ref.npz), against the numpy oracle on seeded random phantoms, on a volume with more
pairs than the first hash table and output array hold, and the key-range check."""

import os

import numpy as np
import pytest

from oracle import decision_points as odp

pytestmark = pytest.mark.gpu

from test_decision_points import CASES, Box3d, assert_equals_fixture, case_args  # noqa: E402


@pytest.fixture(scope='module')
def ref(golden_dir):
  return np.load(os.path.join(golden_dir, 'decision_points_ref.npz'))


def assert_same(got, want):
  assert list(got.keys()) == list(want.keys())
  for key in want:
    assert type(key[0]) is int and type(key[1]) is int
    (dg, pg), (dw, pw) = got[key], want[key]
    assert isinstance(dg, np.float64) and pg.dtype == np.int64 and pg.shape == (3,)
    assert dg == dw, (key, dg, dw)
    assert np.array_equal(pg, pw), (key, pg, pw)


@pytest.mark.parametrize('case', CASES)
def test_device_equals_reference(ref, case):
  from ffn_b200.utils.decision_point import find_decision_points
  seg, kw = case_args(ref, case)
  got = find_decision_points(seg, **kw)
  assert_equals_fixture(ref, case, got, seg)


def test_device_takes_bounding_box_and_any_integer_dtype(ref):
  from ffn_b200.utils.bounding_box import BoundingBox
  from ffn_b200.utils.decision_point import find_decision_points
  seg, kw = case_args(ref, 'aniso_box')
  kw['subvol_box'] = BoundingBox(start=kw['subvol_box'].start, size=kw['subvol_box'].size)
  assert_equals_fixture(ref, 'aniso_box', find_decision_points(seg, **kw), seg)
  # int32 labels, cleared in place
  seg = ref['ut_sparse_opt3_seg'].astype(np.int32)
  assert find_decision_points(seg, (1, 1, 1), optimize_sparse=True, sparse_noise_threshold=3) == {}
  assert np.array_equal(seg, ref['ut_sparse_opt3_seg_after'].astype(np.int32))


def random_phantom(shape, seed, n_boxes):
  """Random boxes of scattered ids (including ids >= 2^63) on a background of 0."""
  rng = np.random.RandomState(seed)
  seg = np.zeros(shape, dtype=np.uint64)
  ids = np.concatenate([rng.randint(1, 50, size=n_boxes // 2).astype(np.uint64),
                        rng.randint(0, 2**62, size=n_boxes - n_boxes // 2).astype(np.uint64) + np.uint64(2**63)])
  for i in ids:
    lo = [rng.randint(0, n) for n in shape]
    hi = [min(n, l + rng.randint(1, max(2, n // 3))) for l, n in zip(lo, shape)]
    seg[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = i
  return seg


PHANTOMS = [
    # shape, seed, boxes, voxel size xyz, max_distance, box (start xyz, size xyz)
    ((17, 23, 29), 1, 12, (1, 1, 1), None, None),
    ((17, 23, 29), 2, 12, (3, 5, 7), 9.5, None),
    ((1, 31, 45), 3, 9, (2, 2, 9), None, ((3, 4, 0), (37, 20, 1))),
    ((13, 1, 27), 4, 7, (1, 1, 1), 3.0, None),
    ((21, 19, 1), 5, 7, (4, 4, 40), None, None),
    ((25, 33, 31), 6, 20, (8, 8, 30), 70.0, ((2, 5, 3), (27, 21, 19))),
]


@pytest.mark.parametrize('shape, seed, n_boxes, voxel_size, max_distance, box', PHANTOMS)
def test_device_equals_oracle(shape, seed, n_boxes, voxel_size, max_distance, box):
  from ffn_b200.utils.decision_point import find_decision_points
  seg = random_phantom(shape, seed, n_boxes)
  kw = dict(max_distance=max_distance, subvol_box=Box3d(*box) if box else None)
  want = odp.find_decision_points(seg.copy(), voxel_size, **kw)
  got = find_decision_points(seg, voxel_size, **kw)
  assert len(want) > 0
  assert_same(got, want)


def test_many_objects_grow_table_and_output():
  """About 6 000 touching Voronoi cells: far more pairs than the first hash table (4096 slots) and the first output
  array hold, so both are enlarged and nothing is dropped."""
  from scipy.spatial import cKDTree
  from ffn_b200.utils import decision_point as dp
  shape = (24, 120, 120)
  sites = np.random.RandomState(31).rand(6000, 3) * np.asarray(shape)
  _, cell = cKDTree(sites).query(np.indices(shape).reshape(3, -1).T.astype(np.float64))
  seg = (cell.reshape(shape).astype(np.uint64) + np.uint64(1)) * np.uint64(2**40) + np.uint64(5)
  assert np.unique(seg).size >= 5000
  want = odp.find_decision_points(seg.copy(), (1, 1, 1))
  got = dp.find_decision_points(seg, (1, 1, 1))
  assert len(want) > 4 * dp._INITIAL_CAP
  assert_same(got, want)


def test_key_range_is_checked():
  from ffn_b200.utils.decision_point import find_decision_points
  seg = np.zeros((3, 3, 3), dtype=np.uint64)
  seg[0, 0, 0], seg[2, 2, 2] = 1, 2
  with pytest.raises(RuntimeError, match='64 bits'):
    find_decision_points(seg, (2**31 - 1, 1, 1))
  assert list(find_decision_points(seg, (2**29, 1, 1))) == [(1, 2)]
