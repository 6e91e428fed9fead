"""Training coordinates without TensorFlow: the GZIP TFRecord files build_coordinates.py writes (inputs.py's
load_patch_coordinates reads them in the reference), parsed as tf.train.Example {center: int64 [x, y, z],
label_volume_name: bytes}.
"""

from __future__ import annotations

import glob as _glob
import gzip
import struct

import numpy as np


def _varint(buf, pos):
  out = shift = 0
  while True:
    b = buf[pos]
    pos += 1
    out |= (b & 0x7F) << shift
    shift += 7
    if b < 0x80:
      return out, pos


def _fields(buf):
  """(field number, wire type, value) of one protobuf message; value is an int (varint) or a bytes slice."""
  pos = 0
  while pos < len(buf):
    key, pos = _varint(buf, pos)
    field, wire = key >> 3, key & 7
    if wire == 0:
      v, pos = _varint(buf, pos)
    elif wire == 2:
      n, pos = _varint(buf, pos)
      v = buf[pos:pos + n]
      pos += n
    elif wire == 1:
      v = buf[pos:pos + 8]
      pos += 8
    elif wire == 5:
      v = buf[pos:pos + 4]
      pos += 4
    else:
      raise ValueError('unsupported protobuf wire type %d' % wire)
    yield field, wire, v


def _feature(buf):
  """A tf.train.Feature as ('bytes', [bytes]) or ('int64', [int])."""
  for field, _, v in _fields(buf):
    if field == 1:
      return 'bytes', [bytes(x) for f, w, x in _fields(v) if f == 1]
    if field == 3:
      vals = []
      for f, w, x in _fields(v):
        if f != 1:
          continue
        if w == 0:
          vals.append(x)
        else:   # packed
          p = 0
          while p < len(x):
            u, p = _varint(x, p)
            vals.append(u)
      return 'int64', [u - (1 << 64) if u >= 1 << 63 else u for u in vals]
    if field == 2:
      return 'float', list(struct.unpack('<%df' % (len(v) // 4), v))
  return 'empty', []


def parse_example(buf) -> dict:
  """tf.train.Example -> {name: (kind, values)}."""
  out = {}
  for field, _, features in _fields(memoryview(buf)):
    if field != 1:
      continue
    for f, _, entry in _fields(features):
      if f != 1:
        continue
      key = value = None
      for ef, _, ev in _fields(entry):
        if ef == 1:
          key = bytes(ev).decode('utf-8')
        elif ef == 2:
          value = _feature(ev)
      out[key] = value if value is not None else ('empty', [])
  return out


def read_records(path):
  """The records of one GZIP TFRecord file (length, masked CRC, data, masked CRC frames)."""
  with gzip.open(path, 'rb') as f:
    data = f.read()
  pos, out = 0, []
  while pos < len(data):
    if pos + 12 > len(data):
      raise ValueError('%s: truncated TFRecord frame header' % path)
    (n,) = struct.unpack_from('<Q', data, pos)
    pos += 12
    if pos + n + 4 > len(data):
      raise ValueError('%s: truncated TFRecord frame' % path)
    out.append(data[pos:pos + n])
    pos += n + 4
  return out


def load_coordinates(pattern: str):
  """Every record of the files matching `pattern` (sorted), in file order: (centers [n, 3] int64 (x, y, z),
  label volume names [n] as str)."""
  paths = sorted(_glob.glob(pattern))
  if not paths:
    raise FileNotFoundError('no coordinate files match %r' % (pattern,))
  centers, names = [], []
  for path in paths:
    for rec in read_records(path):
      ex = parse_example(rec)
      kind_c, center = ex.get('center', ('empty', []))
      kind_n, name = ex.get('label_volume_name', ('empty', []))
      if kind_c != 'int64' or len(center) != 3 or kind_n != 'bytes' or len(name) != 1:
        raise ValueError('%s: a record is not tf.train.Example {center: int64 x 3, label_volume_name: bytes}' % path)
      centers.append(center)
      names.append(name[0].decode('utf-8'))
  return np.array(centers, np.int64).reshape(-1, 3), names
