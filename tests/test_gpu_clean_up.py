"""Connected-component clean-up on the device (ffn_clean_up): against the reference's own clean_up /
clean_up_and_count (tests/golden/clean_up_ref.npz), against the scipy oracle on Voronoi phantoms, on shapes that
stress the union-find (a serpentine, one id filling the volume, salt noise), and through the table-capacity retry."""

import ctypes as C

import numpy as np
import pytest

from ffn_b200 import _lib
from ffn_b200 import synthetic
from ffn_b200.inference import segmentation
from oracle import clean_up as ocu

pytestmark = pytest.mark.gpu

from test_clean_up import CASES, ERRORS, call, check_result  # noqa: E402


@pytest.mark.parametrize('case', CASES, ids=lambda c: c['tag'])
def test_device_equals_reference(case):
  seg = case['seg'].copy()
  if case['error']:
    with pytest.raises(ERRORS[case['error']]):
      call(segmentation, case, seg)
    return
  check_result(case, seg, call(segmentation, case, seg))


def assert_equals_oracle(seg, connectivity, min_size):
  want = seg.copy()
  want_map, want_counts = ocu.clean_up_and_count(want, True, connectivity, min_size)
  got = seg.copy()
  got_map, got_counts = segmentation.clean_up_and_count(got, True, connectivity, min_size)
  assert np.array_equal(got, want), (connectivity, min_size)
  assert got_map == want_map and got_counts == want_counts, (connectivity, min_size)
  assert {type(k) for k in got_map} == {np.uint64} and {type(v) for v in got_map.values()} == {np.uint64}
  assert {type(v) for v in got_counts.values()} == {np.int64}
  return got


@pytest.fixture(scope='module')
def phantom():
  """Voronoi cells with membrane gaps, a cut plane through every cell, and ids above 2^32."""
  _, cells = synthetic.voronoi_phantom((48, 96, 112), seed=5, cell_volume=6000.0, return_cells=True)
  seg = np.where(cells > 0, cells.astype(np.uint64) * np.uint64(2**20) + np.uint64(2**32 + 17), np.uint64(0))
  z, y, x = np.indices(seg.shape)
  seg[(x + 2 * y) % 41 == 0] = 0
  return seg


@pytest.mark.parametrize('connectivity', [1, 2, 3])
@pytest.mark.parametrize('min_size', [0, 30, 1000])
def test_phantom_equals_oracle(phantom, connectivity, min_size):
  got = assert_equals_oracle(phantom, connectivity, min_size)
  assert np.unique(got).size > 50


def test_serpentine_equals_oracle():
  """One id winding through the whole volume: rows joined at alternate ends, planes at alternate corners."""
  sz, sy, sx = 24, 63, 200
  seg = np.zeros((sz, sy, sx), np.uint64)
  for z in range(0, sz, 2):
    seg[z, ::2, :] = 9
    for y in range(1, sy, 2):
      seg[z, y, sx - 1 if (y // 2) % 2 == 0 else 0] = 9
  for z in range(1, sz, 2):
    seg[z, sy - 1 if (z // 2) % 2 == 0 else 0, 0 if (z // 2) % 2 == 0 else sx - 1] = 9
  for c in (1, 3):
    got = assert_equals_oracle(seg, c, 0)
  assert set(np.unique(got)) <= {0, 1}


def test_one_id_fills_the_volume():
  seg = np.full((256, 256, 256), 2**40 + 3, np.uint64)
  id_map, counts = segmentation.clean_up_and_count(seg, connectivity=3)
  assert (seg == 1).all()
  assert id_map == {1: 2**40 + 3} and counts == {1: 256**3}
  seg[...] = 7
  assert segmentation.clean_up(seg, min_size=256**3 + 1, return_id_map=True) == {0: 7}
  assert not seg.any()


@pytest.mark.parametrize('connectivity', [1, 3])
def test_salt_noise_equals_oracle(connectivity):
  """Many small ids: nearly every component is one voxel, and min_size 2 clears them."""
  rng = np.random.RandomState(7)
  seg = rng.randint(1, 10**6, (40, 64, 64)).astype(np.uint64)
  seg[rng.rand(*seg.shape) < 0.2] = 0
  assert_equals_oracle(seg, connectivity, 2)
  got = seg.copy()
  id_map, counts = segmentation.clean_up_and_count(got, connectivity=connectivity, min_size=10)
  assert not got.any() and list(id_map) == [0] and counts == {0: seg.size}


def test_table_capacity_retry():
  """A table larger than the capacity writes nothing; the same call with the reported size succeeds."""
  rng = np.random.RandomState(3)
  seg = rng.randint(0, 3, (20, 30, 40)).astype(np.uint64)
  want = seg.copy()
  want_map, want_counts = ocu.clean_up_and_count(want, True, 1, 2)
  lib = _lib.load()
  desc = _lib.CleanUpDesc(_lib.i3(seg.shape), 1, 2)
  work = seg.copy()
  n_ids = C.c_int64(0)
  cap = 5
  ids, orig, counts = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64), np.zeros(cap, np.int64)
  _lib.check(lib.ffn_clean_up(0, C.byref(desc), _lib.ptr(work), _lib.ptr(ids), _lib.ptr(orig), _lib.ptr(counts), cap,
                              C.byref(n_ids)))
  assert n_ids.value == len(want_map) > cap
  assert np.array_equal(work, seg) and not ids.any() and not counts.any()
  cap = n_ids.value
  ids, orig, counts = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64), np.zeros(cap, np.int64)
  _lib.check(lib.ffn_clean_up(0, C.byref(desc), _lib.ptr(work), _lib.ptr(ids), _lib.ptr(orig), _lib.ptr(counts), cap,
                              C.byref(n_ids)))
  assert n_ids.value == cap and np.array_equal(work, want)
  assert dict(zip(ids, orig)) == want_map and dict(zip(ids, counts)) == want_counts
  # through the host function, whose first capacity is smaller than this table
  big = rng.randint(1, 2**40, (64, 64, 64)).astype(np.uint64)
  assert segmentation.clean_up_and_count(big.copy(), min_size=0)[1] == ocu.clean_up_and_count(big.copy())[1]


def test_bad_arguments_fail_in_the_library():
  lib = _lib.load()
  seg = np.ones((2, 2, 2), np.uint64)
  n_ids = C.c_int64(0)
  # the last extents multiply to 2^64, which wraps to 0 in 64-bit arithmetic
  for shape, conn in (((2, 2, 2), 0), ((2, 2, 2), 4), ((2, -2, 2), 1), ((2**11, 2**10, 2**10), 1),
                      ((2**21, 2**21, 2**22), 1), ((2**30, 2**30, 3), 1)):
    desc = _lib.CleanUpDesc(_lib.i3(shape), conn, 0)
    with pytest.raises(RuntimeError, match='2\\^31|connectivity|negative'):
      _lib.check(lib.ffn_clean_up(0, C.byref(desc), _lib.ptr(seg), None, None, None, 0, C.byref(n_ids)))
  # an empty volume is empty whatever its other extents
  desc = _lib.CleanUpDesc(_lib.i3((2**30, 2**30, 0)), 1, 0)
  n_ids.value = 5
  _lib.check(lib.ffn_clean_up(0, C.byref(desc), None, None, None, None, 0, C.byref(n_ids)))
  assert n_ids.value == 0


def test_non_contiguous_input_is_written_back():
  case = {c['tag']: c for c in CASES}['pieces_c2']
  buf = np.zeros(case['seg'].shape[:2] + (2 * case['seg'].shape[2],), np.uint64)
  view = buf[:, :, ::2]
  view[...] = case['seg']
  check_result(case, view, call(segmentation, case, view))
  assert not buf[:, :, 1::2].any()
