"""Training coordinates from partition maps: build_coordinates (build_coordinates.py:61-112).

Every voxel of a partition volume's crop (the volume without `margin` voxels on each side) whose partition is not 255
becomes a row (volume, flat crop index).  The rows of each partition are permuted and repeated cyclically up to the
size of the largest partition, all of them are shuffled, and each becomes one TFRecord of
tf.train.Example {center: [x, y, z], label_volume_name: name} in one GZIP file, which is what the training input
pipeline reads.

The device splits each crop into its partitions (ffn_partition_rows) and writes the TFRecord frames
(ffn_coordinate_records); there is no host fallback.  The permutations and the shuffle stay on the host and draw from
numpy's global RandomState with the reference's calls, so `np.random.seed(s)` before a call fixes its output and
leaves the generator where the reference leaves it.
"""

from __future__ import annotations

import collections
import ctypes as C
import numbers
import struct
import zlib

import numpy as np

from ffn_b200 import _lib
from ffn_b200.inference import storage

IGNORE_PARTITION = 255
GZIP_LEVEL = 6   # TFRecordWriter's GZIP default, zlib's Z_DEFAULT_COMPRESSION
CHUNK_ROWS = 1 << 20
# zlib's gzip header with no name and no time, as TFRecordWriter's GZIP stream starts.
_GZIP_HEADER = b'\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\x03'
_MAX_PENDING_PIECES = 64


def _margin(margin_zyx):
  m = tuple(margin_zyx)
  if len(m) != 3:
    raise ValueError('margin must have 3 components (z, y, x), got %r' % (margin_zyx,))
  for v in m:
    if not isinstance(v, numbers.Integral) or isinstance(v, bool):
      raise TypeError('margin must hold integers, got %r' % (margin_zyx,))
    if v < 0:
      raise ValueError('margin must not be negative, got %r' % (margin_zyx,))
  return tuple(int(v) for v in m)


def _volume(volume):
  if not isinstance(volume, np.ndarray) or volume.dtype != np.uint8:
    raise TypeError('partition volumes must be uint8 numpy arrays (what compute_partitions writes), got %s'
                    % getattr(volume, 'dtype', type(volume)))
  if volume.ndim != 3:
    raise ValueError('partition volumes must be 3-d, got shape %r' % (volume.shape,))
  return volume


def crop_box(shape, margin_zyx):
  """(start, extent) of volume[mz:-mz, my:-my, mx:-mx], with Python's slice semantics: a margin of 0 is empty."""
  ranges = [range(s)[m:-m] for s, m in zip(shape, margin_zyx)]
  return tuple(r.start if len(r) else 0 for r in ranges), tuple(len(r) for r in ranges)


def partition_rows(volume, margin_zyx, volume_index=0, device=0):
  """The crop's (volume_index, flat index) int64 rows of every partition but 255, grouped by value and in ascending
  flat order within a value, and the crop's 256-bin histogram (int64)."""
  volume = _volume(volume)
  margin = _margin(margin_zyx)
  start, extent = crop_box(volume.shape, margin)
  n = int(np.prod(extent, dtype=np.int64))
  if n >= 2**31:
    raise ValueError('partition crops must have fewer than 2^31 voxels, got %r' % (extent,))
  volume = np.ascontiguousarray(volume)
  rows = np.empty((n, 2), np.int64)
  counts = np.zeros(256, np.int64)
  desc = _lib.PartitionRowsDesc()
  desc.shape_zyx[:] = volume.shape
  desc.crop_start_zyx[:] = start
  desc.crop_shape_zyx[:] = extent
  desc.volume_index = int(volume_index)
  lib = _lib.load()
  _lib.check(lib.ffn_partition_rows(int(device), C.byref(desc), _lib.ptr(volume), _lib.ptr(rows), _lib.ptr(counts)))
  return rows[:n - counts[IGNORE_PARTITION]], counts


def _v16(rows):
  """(n, 2) int64 rows as a 1-d array of n 16-byte items (same memory)."""
  return np.ascontiguousarray(rows, np.int64).reshape(-1, 2).view('V16').reshape(-1)


def resample_and_shuffle(partitions):
  """The reference's resampling on numpy's global RandomState: each (n, 2) int64 array of `partitions` is permuted
  and repeated cyclically to the largest n, the results are concatenated in order and shuffled.

  np.random.permutation and np.random.shuffle draw the same swaps for n 16-byte items as for the n rows of an (n, 2)
  array, but the 1-d call takes numpy's compiled loop instead of a Python loop over rows.  Raises ValueError when
  `partitions` is empty, as the reference's max() does.
  """
  max_count = max(len(p) for p in partitions)
  out = np.empty(max_count * len(partitions), 'V16')
  for k, p in enumerate(partitions):
    perm = np.random.permutation(_v16(p))
    dst = out[k * max_count:(k + 1) * max_count]
    for off in range(0, max_count, len(perm)):   # np.resize: repeat cyclically
      dst[off:off + len(perm)] = perm[:max_count - off]
  np.random.shuffle(out)
  return out.view(np.int64).reshape(-1, 2)


def coordinate_rows(volumes, margin_zyx, device=0):
  """Shuffled (volume, flat crop index) rows of `volumes` (uint8 arrays) and each volume's crop extent."""
  margin = _margin(margin_zyx)
  for v in volumes:
    _volume(v)
  by_value = collections.OrderedDict()   # partitions in the order in which they are first seen
  extents = []
  for i, vol in enumerate(volumes):
    extents.append(crop_box(vol.shape, margin)[1])
    rows, counts = partition_rows(vol, margin, i, device)
    ends = np.cumsum(counts)
    for v in np.flatnonzero(counts[:IGNORE_PARTITION]):
      by_value.setdefault(int(v), []).append(rows[ends[v] - counts[v]:ends[v]])
  partitions = [parts[0] if len(parts) == 1 else np.concatenate(parts) for parts in by_value.values()]
  return resample_and_shuffle(partitions), extents


class GzipMemberWriter:
  """One gzip member written as it is produced: pieces of 4 MB are raw-deflated on storage's thread pool
  (storage._deflate_piece) and written in order; the pieces concatenate to one deflate stream."""

  def __init__(self, fd, level=GZIP_LEVEL):
    self._fd = fd
    self._level = level
    self._crc = 0
    self._size = 0
    self._pending = collections.deque()
    fd.write(_GZIP_HEADER)

  def write(self, data):
    view = memoryview(data).cast('B')
    self._crc = zlib.crc32(view, self._crc)
    self._size += len(view)
    pool = storage._pool()
    for off in range(0, len(view), storage._DEFLATE_CHUNK):
      self._pending.append(pool.submit(storage._deflate_piece, view[off:off + storage._DEFLATE_CHUNK], self._level,
                                       False))
    while len(self._pending) > _MAX_PENDING_PIECES or (self._pending and self._pending[0].done()):
      self._fd.write(self._pending.popleft().result())

  def close(self):
    while self._pending:
      self._fd.write(self._pending.popleft().result())
    self._fd.write(storage._deflate_piece(b'', self._level, True))
    self._fd.write(struct.pack('<II', self._crc & 0xFFFFFFFF, self._size & 0xFFFFFFFF))


def _record_table(names, extents, margin):
  """FfnCoordinateVolume[] and the names blob (UTF-8)."""
  encoded = [n.encode('utf-8') for n in names]
  table = (_lib.CoordinateVolume * max(len(names), 1))()
  off = 0
  for i, (e, ext) in enumerate(zip(encoded, extents)):
    table[i].crop_shape_zyx[:] = ext
    table[i].margin_zyx[:] = margin
    table[i].name_offset = off
    table[i].name_length = len(e)
    off += len(e)
  blob = np.frombuffer(b''.join(encoded) or b'\0', np.uint8).copy()
  return table, blob, max((len(e) for e in encoded), default=0)


def write_records(fd, rows, names, extents, margin_zyx, device=0, chunk_rows=CHUNK_ROWS):
  """Writes the GZIP TFRecord file of `rows` (shuffled (volume, flat) int64) to the binary file `fd`, serialising
  `chunk_rows` rows at a time on the device."""
  if chunk_rows < 1:
    raise ValueError('chunk_rows must be positive, got %r' % (chunk_rows,))
  margin = _margin(margin_zyx)
  table, blob, max_name = _record_table(names, extents, margin)
  desc = _lib.CoordinateDesc()
  desc.volumes = C.cast(table, C.c_void_p)
  desc.n_volumes = len(names)
  desc.names = blob.ctypes.data
  desc.names_bytes = blob.size
  per_row = 130 + max_name   # a frame's largest size: 16 B of framing, the Example with 10-byte varints, the name
  rows = np.ascontiguousarray(rows, np.int64)
  lib = _lib.load()
  out = GzipMemberWriter(fd)
  nbytes = C.c_int64(0)
  for start in range(0, len(rows), chunk_rows):
    chunk = rows[start:start + chunk_rows]
    buf = np.empty(len(chunk) * per_row, np.uint8)
    _lib.check(lib.ffn_coordinate_records(int(device), C.byref(desc), _lib.ptr(chunk), len(chunk), _lib.ptr(buf),
                                          buf.size, C.byref(nbytes)))
    out.write(buf[:nbytes.value])
  out.close()


def build_coordinates(partition_volumes, margin_zyx, coordinate_output, device=0, chunk_rows=CHUNK_ROWS):
  """Builds the GZIP TFRecord file of training coordinates (build_coordinates.py:61-112).

  Args:
    partition_volumes: list of (name, uint8 [z, y, x] partition volume), as compute_partitions writes them; `name`
      is the label_volume_name the trainer looks the volume up by
    margin_zyx: (z, y, x) voxels at each border of every volume that are never sampled, normally the radius of the
      training FoV; 0 on an axis leaves nothing, as the reference's `[m:-m]` crop does
    coordinate_output: path of the GZIP TFRecord file
    device: CUDA device index (an H100)
    chunk_rows: records serialised per device call; the file does not depend on it

  Draws from numpy's global RandomState as the reference does.

  Raises:
    TypeError: for a volume that is not a uint8 array, or a non-integer margin
    ValueError: for a volume that is not 3-d, a crop of 2^31 or more voxels, a negative margin (the reference would
      write centers outside the crop), or when no crop holds a partition other than 255 (as in the reference, before
      the file is created)
  """
  names = [str(n) for n, _ in partition_volumes]
  volumes = [v for _, v in partition_volumes]
  margin = _margin(margin_zyx)
  for v in volumes:
    n = int(np.prod(crop_box(_volume(v).shape, margin)[1], dtype=np.int64))
    if n >= 2**31:
      raise ValueError('partition crops must have fewer than 2^31 voxels, got %d' % n)
  rows, extents = coordinate_rows(volumes, margin, device)
  with open(coordinate_output, 'wb') as fd:
    write_records(fd, rows, names, extents, margin, device, chunk_rows)
