"""Training coordinates (build_coordinates.py:61-112): the numpy oracle against the reference's own script
(tests/golden/coordinates_ref.npz, from make_golden_coordinates.py), the host shuffle against the oracle's, the gzip
assembly, a TFRecord reader with its CRC-32C and Example descriptor, and the argument checks of
ffn_b200.coordinates and of the build_coordinates.py script, none of which needs a device."""

import gzip
import io
import os
import struct

import numpy as np
import pytest
from google.protobuf import descriptor_pb2
from google.protobuf import descriptor_pool
from google.protobuf import message_factory

import build_coordinates as script
from ffn_b200 import coordinates
from oracle import coordinates as oc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'coordinates_ref.npz')
ERRORS = {'ValueError': ValueError}


def fixture():
  return np.load(GOLDEN)


def reference_cases():
  """One dict per fixture case: the named volumes, margin, seed, number of `main` calls after the seed, and per
  call the records' centers (x, y, z) and name indices, or the name of the exception."""
  g = fixture()
  out = []
  for i in range(int(g['n_cases'])):
    names = [str(n) for n in g['names_%d' % i]]
    calls, error = int(g['calls_%d' % i]), str(g['error_%d' % i])
    out.append({
        'tag': str(g['tag_%d' % i]),
        'volumes': [(names[k], g['volume_%d_%d' % (i, k)]) for k in range(int(g['n_volumes_%d' % i]))],
        'margin': tuple(int(m) for m in g['margin_%d' % i]), 'seed': int(g['seed_%d' % i]), 'calls': calls,
        'error': error,
        'centers': [] if error else [g['centers_%d_%d' % (i, c)].astype(np.int64) for c in range(calls)],
        'name_index': [] if error else [g['name_index_%d_%d' % (i, c)].astype(np.int64) for c in range(calls)]})
  return out


def case_ids():
  g = fixture()
  return [str(g['tag_%d' % i]) for i in range(int(g['n_cases']))]


# ---- test-local TFRecord reader ---------------------------------------------------------------------------------

def _crc32c_table():
  t = np.zeros(256, np.uint32)
  for i in range(256):
    c = i
    for _ in range(8):
      c = (c >> 1) ^ (0x82F63B78 if c & 1 else 0)
    t[i] = c
  return t


_CRC32C = _crc32c_table()


def crc32c_rows(data):
  """CRC-32C (Castagnoli, reflected) of every row of a (m, n) uint8 array."""
  crc = np.full(data.shape[0], 0xFFFFFFFF, np.uint32)
  for j in range(data.shape[1]):
    crc = _CRC32C[(crc ^ data[:, j]) & 0xFF] ^ (crc >> np.uint32(8))
  return crc ^ np.uint32(0xFFFFFFFF)


def crc32c(data):
  return int(crc32c_rows(np.frombuffer(bytes(data), np.uint8)[None])[0])


def masked(crc):
  crc = crc.astype(np.uint64)
  return ((((crc >> np.uint64(15)) | (crc << np.uint64(17))) + np.uint64(0xa282ead8)) & np.uint64(0xFFFFFFFF))


def tfrecord_payloads(raw):
  """The payloads of uncompressed TFRecord bytes, with both CRCs of every frame checked."""
  offs, lens = [], []
  off = 0
  while off < len(raw):
    assert off + 12 <= len(raw), 'truncated frame header'
    n = struct.unpack_from('<Q', raw, off)[0]
    offs.append(off)
    lens.append(n)
    off += 16 + n
  assert off == len(raw), 'truncated frame'
  buf = np.frombuffer(raw, np.uint8)
  offs, lens = np.array(offs, np.int64), np.array(lens, np.int64)
  for n in np.unique(lens):
    at = offs[lens == n]
    head = buf[at[:, None] + np.arange(12)]
    assert (masked(crc32c_rows(head[:, :8])) == head[:, 8:12].copy().view('<u4')[:, 0]).all(), 'length CRC'
    body = buf[at[:, None] + 12 + np.arange(n + 4)]
    assert (masked(crc32c_rows(body[:, :n])) == body[:, n:].copy().view('<u4')[:, 0]).all(), 'payload CRC'
  return [raw[o + 12:o + 12 + n] for o, n in zip(offs.tolist(), lens.tolist())]


def example_class():
  """tf.train.Example (tensorflow/core/example/{example,feature}.proto), built at run time in a private pool."""
  f = descriptor_pb2.FileDescriptorProto(name='ffn_test_example.proto', package='tensorflow', syntax='proto3')
  T = descriptor_pb2.FieldDescriptorProto
  rep, opt = T.LABEL_REPEATED, T.LABEL_OPTIONAL

  def msg(name, *fields):
    m = f.message_type.add(name=name)
    for fname, num, typ, label, tname in fields:
      m.field.add(name=fname, number=num, type=typ, label=label, type_name=tname)
    return m
  msg('BytesList', ('value', 1, T.TYPE_BYTES, rep, None))
  msg('FloatList', ('value', 1, T.TYPE_FLOAT, rep, None))
  msg('Int64List', ('value', 1, T.TYPE_INT64, rep, None))
  feat = msg('Feature', ('bytes_list', 1, T.TYPE_MESSAGE, opt, '.tensorflow.BytesList'),
             ('float_list', 2, T.TYPE_MESSAGE, opt, '.tensorflow.FloatList'),
             ('int64_list', 3, T.TYPE_MESSAGE, opt, '.tensorflow.Int64List'))
  feat.oneof_decl.add(name='kind')
  for fld in feat.field:
    fld.oneof_index = 0
  feats = msg('Features', ('feature', 1, T.TYPE_MESSAGE, rep, '.tensorflow.Features.FeatureEntry'))
  entry = feats.nested_type.add(name='FeatureEntry')
  entry.options.map_entry = True
  entry.field.add(name='key', number=1, type=T.TYPE_STRING, label=opt)
  entry.field.add(name='value', number=2, type=T.TYPE_MESSAGE, label=opt, type_name='.tensorflow.Feature')
  msg('Example', ('features', 1, T.TYPE_MESSAGE, opt, '.tensorflow.Features'))
  pool = descriptor_pool.DescriptorPool()
  pool.Add(f)
  return message_factory.GetMessageClass(pool.FindMessageTypeByName('tensorflow.Example'))


def read_coordinates(path):
  """(centers (n, 3) int64, names [bytes]) of a GZIP TFRecord file of coordinate Examples; every payload must be
  the deterministic serialisation of the Example it parses to."""
  with open(path, 'rb') as f:
    raw = gzip.decompress(f.read())
  Example = example_class()
  centers, names = [], []
  for p in tfrecord_payloads(raw):
    ex = Example.FromString(p)
    assert sorted(ex.features.feature) == ['center', 'label_volume_name']
    c = ex.features.feature['center']
    n = ex.features.feature['label_volume_name']
    assert c.WhichOneof('kind') == 'int64_list' and n.WhichOneof('kind') == 'bytes_list'
    assert len(c.int64_list.value) == 3 and len(n.bytes_list.value) == 1
    assert ex.SerializeToString(deterministic=True) == p
    centers.append(list(c.int64_list.value))
    names.append(n.bytes_list.value[0])
  return np.array(centers, np.int64).reshape(-1, 3), names


# ---- tests ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('idx', range(len(case_ids())), ids=case_ids())
def test_oracle_equals_reference(idx):
  c = reference_cases()[idx]
  arrays = [v for _, v in c['volumes']]
  np.random.seed(c['seed'])
  if c['error']:
    with pytest.raises(ERRORS[c['error']]):
      oc.build_coordinates(arrays, c['margin'])
    return
  for k in range(c['calls']):
    centers, vol = oc.build_coordinates(arrays, c['margin'])
    assert centers.shape == c['centers'][k].shape and (centers == c['centers'][k]).all()
    assert (vol == c['name_index'][k]).all()


def host_buckets(volumes, margin):
  """What the device bucketing returns, from np.flatnonzero: per partition in first-seen order, its rows."""
  parts = {}
  for i, vol in enumerate(volumes):
    crop = vol[margin[0]:-margin[0], margin[1]:-margin[1], margin[2]:-margin[2]]
    for v in range(255):
      flat = np.flatnonzero(crop == v)
      if flat.size:
        parts.setdefault(v, []).append(np.stack([np.full(flat.size, i), flat], 1).astype(np.int64))
  return [np.concatenate(p) for p in parts.values()]


@pytest.mark.parametrize('seed', [0, 1, 2018])
@pytest.mark.parametrize('shapes', [[(3, 3, 3)], [(9, 10, 11)], [(20, 30, 25), (12, 40, 9)]], ids=str)
def test_host_shuffle_equals_oracle(seed, shapes):
  rng = np.random.RandomState(seed + 100)
  volumes = [(rng.zipf(1.6, s) % 7 * 37).astype(np.uint8) for s in shapes]
  volumes[0].flat[0] = 255
  np.random.seed(seed)
  want, _ = oc.coordinate_rows(volumes, (1, 1, 1))
  want_state = np.random.get_state()
  np.random.seed(seed)
  got = coordinates.resample_and_shuffle(host_buckets(volumes, (1, 1, 1)))
  got_state = np.random.get_state()
  assert got.dtype == np.int64 and got.shape == want.shape and (got == want).all()
  assert got_state[0] == want_state[0] and (got_state[1] == want_state[1]).all()
  assert got_state[2:] == want_state[2:]


def test_resample_of_nothing_raises():
  with pytest.raises(ValueError):
    coordinates.resample_and_shuffle([])


@pytest.mark.parametrize('sizes', [[100], [0], [9 << 20], [3, 0, 5 << 20, 17, 4 << 20]], ids=str)
def test_gzip_member_decompresses_to_input(sizes):
  rng = np.random.RandomState(1)
  parts = [(rng.zipf(1.3, n) % 251).astype(np.uint8).tobytes() for n in sizes]
  fd = io.BytesIO()
  w = coordinates.GzipMemberWriter(fd)
  for p in parts:
    w.write(p)
  w.close()
  assert gzip.decompress(fd.getvalue()) == b''.join(parts)


def test_crc32c_known_answers():
  # RFC 3720, B.4
  assert crc32c(b'123456789') == 0xE3069283
  assert crc32c(bytes(32)) == 0x8A9136AA


def test_example_descriptor_known_answer():
  Example = example_class()
  ex = Example()
  ex.features.feature['label_volume_name'].bytes_list.value.append(b'vol')
  ex.features.feature['center'].int64_list.value.extend([300, 5, 70000])
  want = bytes.fromhex('0a340a140a0663656e746572120a1a080a06ac0205f0a2040a1c0a116c6162656c5f766f6c756d655f6e616d65'
                       '12070a050a03766f6c')
  assert ex.SerializeToString(deterministic=True) == want


def test_crop_box_is_the_slice():
  for s in (0, 1, 2, 5, 8):
    for m in (0, 1, 2, 3, 4, 9):
      vol = np.zeros((s, 1, 1))
      start, extent = coordinates.crop_box((s, 1, 1), (m, 0, 0))
      assert extent[0] == vol[m:-m].shape[0]
      if extent[0]:
        assert start[0] == m


def test_refusals(tmp_path):
  out = str(tmp_path / 'c.tfrecord.gz')
  good = np.zeros((6, 6, 6), np.uint8)
  with pytest.raises(TypeError):
    coordinates.build_coordinates([('a', good.astype(np.int16))], (1, 1, 1), out)
  with pytest.raises(TypeError):
    coordinates.build_coordinates([('a', good.tolist())], (1, 1, 1), out)
  with pytest.raises(ValueError):
    coordinates.build_coordinates([('a', good[0])], (1, 1, 1), out)
  with pytest.raises(ValueError):
    coordinates.build_coordinates([('a', good)], (1, -1, 1), out)
  with pytest.raises(ValueError):
    coordinates.build_coordinates([('a', good)], (1, 1), out)
  with pytest.raises(TypeError):
    coordinates.build_coordinates([('a', good)], (1, 1.5, 1), out)
  huge = np.broadcast_to(np.uint8(3), (2050, 1026, 1026))   # a 2^31-voxel crop, never materialised
  with pytest.raises(ValueError, match='2\\^31'):
    coordinates.build_coordinates([('a', good), ('b', huge)], (1, 1, 1), out)
  assert not os.path.exists(out)


def test_margin_zero_raises_as_reference(tmp_path):
  # A margin of 0 empties every crop: the reference's max() over no partitions raises before any draw or file.
  out = str(tmp_path / 'c.tfrecord.gz')
  np.random.seed(4)
  state = np.random.get_state()
  with pytest.raises(ValueError):
    coordinates.build_coordinates([('a', np.ones((6, 6, 6), np.uint8))], (0, 1, 1), out)
  assert (np.random.get_state()[1] == state[1]).all() and np.random.get_state()[2] == state[2]
  assert not os.path.exists(out)


@pytest.mark.parametrize('entry', ['vol:path.npz', 'vol:path.npz:af:x', 'vol'])
def test_script_rejects_entries_without_two_colons(entry, tmp_path):
  script.FLAGS(['build_coordinates.py', '--partition_volumes=' + entry, '--margin=1,1,1',
                '--coordinate_output=%s' % (tmp_path / 'c.gz')])
  with pytest.raises(ValueError):
    script.main([])
