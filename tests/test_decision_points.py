"""find_decision_points on the host side: the numpy oracle (oracle/decision_points.py) against the reference's own
function (tests/golden/decision_points_ref.npz) and against the literal expectations of the reference's unit test
(ffn/utils/tests/decision_point_test.py); input validation of the device wrapper; the ffn.utils drop-in path."""

import os

import numpy as np
import pytest

from oracle import decision_points as odp

CASES = ['ut_two', 'ut_three', 'ut_three_md30', 'ut_sparse', 'ut_sparse_opt0', 'ut_sparse_opt3', 'ut_single_opt0',
         'voronoi_gaps', 'voronoi_touch', 'voronoi_dust', 'aniso_box']


class Box3d:
  """A box that only offers to_slice3d (the connectomics BoundingBox interface)."""

  def __init__(self, start_xyz, size_xyz):
    self.start, self.size = np.asarray(start_xyz), np.asarray(size_xyz)

  def to_slice3d(self):
    lo, hi = self.start, self.start + self.size
    return np.index_exp[lo[2]:hi[2], lo[1]:hi[1], lo[0]:hi[0]]


@pytest.fixture(scope='module')
def ref(golden_dir):
  return np.load(os.path.join(golden_dir, 'decision_points_ref.npz'))


def case_args(ref, case):
  """(seg copy, kwargs) of a fixture case."""
  md = float(ref[case + '_max_distance'])
  box = ref[case + '_box']
  return ref[case + '_seg'].copy(), dict(
      voxel_size=tuple(int(v) for v in ref[case + '_voxel_size']),
      max_distance=None if np.isnan(md) else md,
      subvol_box=Box3d(box[:3], box[3:]) if box.size else None,
      optimize_sparse=bool(ref[case + '_optimize_sparse']),
      sparse_noise_threshold=int(ref[case + '_threshold']))


def assert_equals_fixture(ref, case, got, seg_after):
  ids, dist, points = ref[case + '_ids'], ref[case + '_dist'], ref[case + '_points']
  assert list(got.keys()) == [(int(a), int(b)) for a, b in ids]
  for k, (key, (d, p)) in enumerate(got.items()):
    assert d == dist[k], (key, d, dist[k])
    assert np.array_equal(p, points[k]), (key, p, points[k])
  assert np.array_equal(seg_after, ref[case + '_seg_after'])


def test_fixture_covers_the_issue_cases(ref):
  assert list(ref['cases']) == CASES
  big = ref['voronoi_gaps_ids']
  assert (big >= np.uint64(2**63)).any() and ((big >= np.uint64(2**32)) & (big < np.uint64(2**63))).any()
  assert (ref['voronoi_touch_dist'] == 0).any()
  assert not np.array_equal(ref['voronoi_dust_seg'], ref['voronoi_dust_seg_after'])


@pytest.mark.parametrize('case', CASES)
def test_oracle_equals_reference(ref, case):
  seg, kw = case_args(ref, case)
  got = odp.find_decision_points(seg, **kw)
  assert_equals_fixture(ref, case, got, seg)


def test_oracle_reference_unit_test_expectations():
  seg = np.zeros((100, 80, 60), dtype=np.uint64)
  seg[:40] = 1
  seg[60:] = 2
  points = odp.find_decision_points(seg, (1, 1, 1))
  assert list(points) == [(1, 2)]
  assert points[(1, 2)][0] == 10 and points[(1, 2)][1].tolist() == [29, 39, 49]

  seg = np.zeros((1, 100, 100), dtype=np.uint64)
  seg[0, :20, :20] = 1
  seg[0, :20:, -20:] = 2
  seg[0, -20:, 40:60] = 3
  points = odp.find_decision_points(seg, (1, 1, 1))
  assert sorted(points) == [(1, 2), (1, 3), (2, 3)]
  assert points[(1, 2)][1].tolist() == [49, 9, 0]
  assert points[(1, 3)][1].tolist() == [29, 49, 0]
  assert points[(2, 3)][1].tolist() == [69, 49, 0]
  assert list(odp.find_decision_points(seg, (1, 1, 1), max_distance=30.0)) == [(1, 2)]

  seg = np.zeros((100, 80, 60), dtype=np.uint64)
  seg[:40] = 1
  seg[60, 0, 0] = seg[61, 0, 0] = 2
  assert (1, 2) in odp.find_decision_points(seg.copy(), (1, 1, 1))
  assert (1, 2) in odp.find_decision_points(seg.copy(), (1, 1, 1), optimize_sparse=True, sparse_noise_threshold=0)
  assert odp.find_decision_points(seg, (1, 1, 1), optimize_sparse=True, sparse_noise_threshold=3) == {}
  assert not (seg == 2).any()   # cleared in place

  seg = np.zeros((100, 80, 60), dtype=np.uint64)
  seg[:40] = 1
  assert odp.find_decision_points(seg, (1, 1, 1), optimize_sparse=True, sparse_noise_threshold=0) == {}


def test_oracle_smallest_id_wins_ties():
  seg = np.zeros((1, 1, 5), dtype=np.uint64)
  seg[0, 0, 0], seg[0, 0, 4] = 7, 3
  expanded, edt = odp.watershed_expand(seg, (1, 1, 1))
  assert expanded[0, 0].tolist() == [7, 7, 3, 3, 3]
  assert edt[0, 0].tolist() == [0, 1, 2, 1, 0]


@pytest.mark.parametrize('kwargs, match', [
    ({'voxel_size': (8.5, 8, 30)}, 'positive integers'),
    ({'voxel_size': (0, 1, 1)}, 'positive integers'),
    ({'voxel_size': (-4, 1, 1)}, 'positive integers'),
    ({'voxel_size': (1, 1)}, '3 components'),
    ({'voxel_size': (1, 1, 1), 'subvol_box': Box3d((0, 0, 0), (7, 6, 6))}, 'outside'),
    ({'voxel_size': (1, 1, 1), 'subvol_box': Box3d((-1, 0, 0), (2, 2, 2))}, 'outside'),
])
def test_wrapper_rejects_bad_arguments(kwargs, match):
  from ffn_b200.utils.bounding_box import BoundingBox
  from ffn_b200.utils.decision_point import find_decision_points
  seg = np.zeros((5, 6, 6), dtype=np.uint64)
  seg[1, 1, 1], seg[3, 4, 4] = 1, 2
  with pytest.raises(ValueError, match=match):
    find_decision_points(seg, **kwargs)
  with pytest.raises(ValueError, match='outside'):
    find_decision_points(seg, (1, 1, 1), subvol_box=BoundingBox(start=(0, 0, 4), size=(6, 6, 2)))


def test_wrapper_rejects_bad_labels():
  from ffn_b200.utils.decision_point import find_decision_points
  seg = np.zeros((4, 4, 4), dtype=np.int32)
  seg[0, 0, 0] = -1
  with pytest.raises(ValueError, match='negative'):
    find_decision_points(seg, (1, 1, 1))
  with pytest.raises(ValueError, match='integer'):
    find_decision_points(np.zeros((4, 4, 4), dtype=np.float32), (1, 1, 1))
  with pytest.raises(ValueError, match='3d'):
    find_decision_points(np.zeros((4, 4), dtype=np.uint64), (1, 1, 1))


def test_drop_in_module():
  from ffn.utils import decision_point
  from ffn_b200.utils import decision_point as impl
  assert decision_point is impl
  assert decision_point.find_decision_points is impl.find_decision_points


def test_no_host_fallback():
  import torch
  if torch.cuda.is_available():
    pytest.skip('a CUDA device is present')
  from ffn_b200.utils.decision_point import find_decision_points
  seg = np.zeros((4, 4, 4), dtype=np.uint64)
  seg[0], seg[3] = 1, 2
  with pytest.raises(RuntimeError, match='CUDA device'):
    find_decision_points(seg, (1, 1, 1))
