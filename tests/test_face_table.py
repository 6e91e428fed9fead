"""The table the flood kernel reduces the movement policy's faces from, and the packed (score, index) maximum it is
reduced with (CPU only: the table comes from the library's host code, the key arithmetic is modelled in numpy)."""

import ctypes as C

import numpy as np
import pytest

from ffn_b200 import _lib

TILE_OUT = 126   # FoV rows per tile (kTileOut)

# field of view, deltas: the flood-fill geometries of test_gpu_geometry.py and the FIB-25 model
GEOMETRIES = [((33, 33, 33), (8, 8, 8)), ((9, 17, 25), (2, 4, 6)), ((5, 33, 33), (0, 8, 8)), ((3, 3, 3), (1, 1, 1)),
              ((17, 33, 17), (8, 8, 8)), ((5, 5, 5), (2, 0, 1))]


def _table(fov, deltas):
  lib = _lib.load()
  desc = _lib.ModelDesc()
  desc.fov_zyx = _lib.i3(fov)
  desc.deltas_zyx = _lib.i3(deltas)
  desc.depth, desc.features = 2, 32
  n, nt = C.c_int64(), C.c_int64()
  _lib.check(lib.ffn_face_table(C.byref(desc), 0, None, C.byref(n), None, C.byref(nt)))
  entries = np.zeros((n.value, 3), dtype=np.int32)
  first = np.zeros(nt.value + 1, dtype=np.int32)
  _lib.check(lib.ffn_face_table(C.byref(desc), n.value, entries.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(n),
                                first.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(nt)))
  return entries, first


def _faces(fov, deltas):
  """(row, face, e) of every face voxel as movement.get_scored_move_offsets enumerates them: per axis with a nonzero
  delta the faces at -delta and +delta, the other two axes in C order over [centre - delta, centre + delta]."""
  xp, pp = fov[2], (fov[1] + 1) * fov[2]
  out = []
  for axis in range(3):
    if deltas[axis] == 0:
      continue
    others = [a for a in range(3) if a != axis]
    for side in (0, 1):
      e = 0
      for i0 in range(2 * deltas[others[0]] + 1):
        for i1 in range(2 * deltas[others[1]] + 1):
          zyx = [0, 0, 0]
          zyx[axis] = fov[axis] // 2 + (deltas[axis] if side else -deltas[axis])
          zyx[others[0]] = fov[others[0]] // 2 - deltas[others[0]] + i0
          zyx[others[1]] = fov[others[1]] // 2 - deltas[others[1]] + i1
          out.append((zyx[0] * pp + zyx[1] * xp + zyx[2], 2 * axis + side, e))
          e += 1
  return out


@pytest.mark.parametrize('fov,deltas', GEOMETRIES)
def test_table_lists_the_policy_faces_by_row(fov, deltas):
  entries, first = _table(fov, deltas)
  want = _faces(fov, deltas)
  assert len(want) == sum(2 * np.prod([2 * deltas[a] + 1 for a in range(3) if a != ax]) for ax in range(3) if deltas[ax])
  assert sorted(map(tuple, entries.tolist())) == sorted(want)
  rows = entries[:, 0]
  assert np.all(np.diff(rows) >= 0)
  # every tile finds exactly the entries of its own output rows
  nt = len(first) - 1
  assert first[0] == 0 and first[-1] == len(entries) and rows.max(initial=0) < nt * TILE_OUT
  for t in range(nt):
    sel = rows[first[t]:first[t + 1]]
    assert np.all(sel // TILE_OUT == t)
  assert np.array_equal(np.bincount(rows // TILE_OUT, minlength=nt), np.diff(first))


def _keys(scores, idx):
  """face_key: order-preserving bits of the score (with -0.0 as +0.0) above 0xffffffff - index."""
  s = np.where(scores == 0, np.float32(0), scores).astype(np.float32)
  b = s.view(np.uint32).astype(np.uint64)
  b = np.where(b >> np.uint64(31), b ^ np.uint64(0xffffffff), b ^ np.uint64(0x80000000))
  return (b << np.uint64(32)) | (np.uint64(0xffffffff) - idx.astype(np.uint64))


def _unpack(key):
  b = np.uint64(key) >> np.uint64(32)
  b = b ^ np.uint64(0x80000000) if b >> np.uint64(31) else b ^ np.uint64(0xffffffff)
  return np.array([b], dtype=np.uint64).astype(np.uint32).view(np.float32)[0], int(np.uint64(0xffffffff) - (np.uint64(key) & np.uint64(0xffffffff)))


def test_packed_key_maximum_is_the_first_index_argmax():
  rng = np.random.RandomState(7)
  for trial in range(200):
    n = int(rng.randint(1, 290))
    s = (rng.randn(n) * 10 ** rng.uniform(-3, 2)).astype(np.float32)
    if trial % 2:   # forced ties, among them the maximum
      s[rng.randint(0, n, size=n // 2 + 1)] = s.max()
    if trial % 3 == 0:   # signed zeros that tie with each other
      s = np.minimum(s, np.float32(0))
      z = rng.randint(0, n, size=4)
      s[z] = np.where(rng.rand(4) < 0.5, np.float32(-0.0), np.float32(0.0))
    if trial % 7 == 0:
      s[rng.randint(0, n)] = -np.inf
    order = rng.permutation(n)   # the atomics arrive in any order
    best, best_i = _unpack(_keys(s[order], order).max())
    assert best_i == int(np.argmax(s))
    assert best == s[best_i] and (best != 0 or not np.signbit(best))
