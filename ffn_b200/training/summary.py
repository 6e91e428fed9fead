"""TensorBoard event files without TensorFlow: `Event` / `Summary` messages built from runtime descriptors with the
field numbers of TensorBoard's event.proto and summary.proto, in TFRecord frames with masked CRC-32C checksums.

    w = EventWriter(logdir)           # events.out.tfevents.<time>.<host>, first record file_version "brain.Event:2"
    w.add(step, [('eval/patch_loss', 0.31), ('final_xy/0', tracker.Image(h, w, png))])
    w.close()
"""

from __future__ import annotations

import os
import socket
import struct
import time

from google.protobuf import descriptor_pb2
from google.protobuf import descriptor_pool
from google.protobuf import message_factory

from .tracker import Image

_F = descriptor_pb2.FieldDescriptorProto


def _field(msg, name, number, ftype, type_name=None, repeated=False, oneof=None):
  f = msg.field.add()
  f.name, f.number, f.type = name, number, ftype
  f.label = _F.LABEL_REPEATED if repeated else _F.LABEL_OPTIONAL
  if type_name:
    f.type_name = type_name
  if oneof is not None:
    f.oneof_index = oneof


def _build():
  """tensorflow.Event { wall_time = 1, step = 2, oneof what { file_version = 3, summary = 5 } } and
  tensorflow.Summary { repeated Value value = 1 }, Value { tag = 1, oneof value { simple_value = 2, image = 4 } },
  Image { height = 1, width = 2, colorspace = 3, encoded_image_string = 4 }: the fields this writer uses."""
  fd = descriptor_pb2.FileDescriptorProto(name='ffn_b200/tensorboard_event.proto', package='tensorflow',
                                          syntax='proto3')
  s = fd.message_type.add(name='Summary')
  im = s.nested_type.add(name='Image')
  _field(im, 'height', 1, _F.TYPE_INT32)
  _field(im, 'width', 2, _F.TYPE_INT32)
  _field(im, 'colorspace', 3, _F.TYPE_INT32)
  _field(im, 'encoded_image_string', 4, _F.TYPE_BYTES)
  v = s.nested_type.add(name='Value')
  v.oneof_decl.add(name='value')
  _field(v, 'tag', 1, _F.TYPE_STRING)
  _field(v, 'simple_value', 2, _F.TYPE_FLOAT, oneof=0)
  _field(v, 'image', 4, _F.TYPE_MESSAGE, '.tensorflow.Summary.Image', oneof=0)
  _field(s, 'value', 1, _F.TYPE_MESSAGE, '.tensorflow.Summary.Value', repeated=True)
  e = fd.message_type.add(name='Event')
  e.oneof_decl.add(name='what')
  _field(e, 'wall_time', 1, _F.TYPE_DOUBLE)
  _field(e, 'step', 2, _F.TYPE_INT64)
  _field(e, 'file_version', 3, _F.TYPE_STRING, oneof=0)
  _field(e, 'summary', 5, _F.TYPE_MESSAGE, '.tensorflow.Summary', oneof=0)
  pool = descriptor_pool.DescriptorPool()   # private: never clashes with an installed TensorBoard
  pool.Add(fd)
  f = pool.FindFileByName(fd.name)
  return (message_factory.GetMessageClass(f.message_types_by_name['Event']),
          message_factory.GetMessageClass(f.message_types_by_name['Summary']))


Event, Summary = _build()


def _crc32c_table():
  table = []
  for i in range(256):
    c = i
    for _ in range(8):
      c = (c >> 1) ^ 0x82F63B78 if c & 1 else c >> 1
    table.append(c)
  return table


_CRC_TABLE = _crc32c_table()


def crc32c(data: bytes) -> int:
  """CRC-32C (Castagnoli, reflected polynomial 0x82F63B78), as RFC 3720 defines it."""
  c = 0xFFFFFFFF
  t = _CRC_TABLE
  for b in data:
    c = t[(c ^ b) & 0xFF] ^ (c >> 8)
  return c ^ 0xFFFFFFFF


def masked_crc32c(data: bytes) -> int:
  """TFRecord's masked checksum: the CRC rotated right by 15 bits plus 0xa282ead8."""
  c = crc32c(data)
  return (((c >> 15) | (c << 17)) + 0xA282EAD8) & 0xFFFFFFFF


def frame(data: bytes) -> bytes:
  """One TFRecord: uint64 length, masked CRC of the length, data, masked CRC of the data (little-endian)."""
  n = struct.pack('<Q', len(data))
  return n + struct.pack('<I', masked_crc32c(n)) + data + struct.pack('<I', masked_crc32c(data))


def read_records(path: str) -> list:
  """The records of an uncompressed TFRecord file, each frame's checksums verified."""
  with open(path, 'rb') as f:
    data = f.read()
  pos, out = 0, []
  while pos < len(data):
    if pos + 12 > len(data):
      raise ValueError('%s: truncated TFRecord frame header' % path)
    n_bytes = data[pos:pos + 8]
    (n,) = struct.unpack('<Q', n_bytes)
    (c,) = struct.unpack_from('<I', data, pos + 8)
    if c != masked_crc32c(n_bytes) or pos + 12 + n + 4 > len(data):
      raise ValueError('%s: corrupt TFRecord frame at byte %d' % (path, pos))
    rec = data[pos + 12:pos + 12 + n]
    (c,) = struct.unpack_from('<I', data, pos + 12 + n)
    if c != masked_crc32c(rec):
      raise ValueError('%s: record checksum mismatch at byte %d' % (path, pos))
    out.append(rec)
    pos += 12 + n + 4
  return out


def read_events(path: str) -> list:
  """The Event messages of an event file."""
  out = []
  for rec in read_records(path):
    ev = Event()
    ev.ParseFromString(rec)
    out.append(ev)
  return out


class EventWriter:
  """Appends Event records to events.out.tfevents.<time>.<host> in logdir."""

  def __init__(self, logdir: str):
    os.makedirs(logdir, exist_ok=True)
    now = time.time()
    self.path = os.path.join(logdir, 'events.out.tfevents.%010d.%s' % (int(now), socket.gethostname()))
    self._f = open(self.path, 'ab')
    self._write(Event(wall_time=now, file_version='brain.Event:2'))

  def _write(self, ev):
    self._f.write(frame(ev.SerializeToString()))
    self._f.flush()

  def add(self, step: int, values, wall_time: float | None = None):
    """One Event at `step` holding a Summary of values: [(tag, number or tracker.Image)]."""
    summ = Summary()
    for tag, v in values:
      val = summ.value.add(tag=tag)
      if isinstance(v, Image):
        val.image.height, val.image.width, val.image.colorspace = v.height, v.width, 3
        val.image.encoded_image_string = v.png
      else:
        val.simple_value = float(v)
    self._write(Event(wall_time=time.time() if wall_time is None else wall_time, step=int(step), summary=summ))

  def close(self):
    if self._f:
      self._f.close()
      self._f = None
