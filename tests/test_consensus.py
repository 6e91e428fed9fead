"""Split consensus on the host: the oracle against the fixture written by the reference's own modules
(tests/golden/make_golden_consensus.py), ConsensusRequest against consensus.proto, load_segmentation_from_source, and
the input checks that run before any device work."""
import os

import numpy as np
import pytest

from ffn_b200.inference import consensus_pb2
from ffn_b200.inference import segmentation
from ffn_b200.inference import storage
from oracle import consensus as oc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'consensus_ref.npz')
ERRORS = {'ValueError': ValueError, 'TypeError': TypeError}


def split_cases():
  """(tag, a, b, min_size, type, expected array or None, v1 after the call, expected error name) per case."""
  g = np.load(GOLDEN)
  return [(str(g['tag_%d' % i]), g['a_%d' % i], g['b_%d' % i], int(g['min_size_%d' % i]), int(g['type_%d' % i]),
           g['out_%d' % i], g['v1_after_%d' % i], str(g['error_%d' % i])) for i in range(int(g['n_split']))]


def write_sources(tmp_path):
  """The fixture's two seg-*.npz and .prob under tmp_path; (dir1, dir2, corner)."""
  g = np.load(GOLDEN)
  for name in ('seg1', 'prob1', 'seg2'):
    path = tmp_path / str(g['relpath_' + name])
    path.parent.mkdir(parents=True, exist_ok=True)
    path.write_bytes(g['file_' + name].tobytes())
  return str(tmp_path / 'forward'), str(tmp_path / 'reverse'), tuple(int(v) for v in g['corner'])


def consensus_cases(tmp_path):
  """(tag, request, expected loaded arrays and origin ids, expected segmentation and origins) per case."""
  g = np.load(GOLDEN)
  d1, d2, corner = write_sources(tmp_path)
  out = []
  for i in range(int(g['n_consensus'])):
    req = consensus_pb2.ConsensusRequest(split_min_size=int(g['split_min_size_%d' % i]))
    req.segmentation1.directory = d1
    req.segmentation1.split_cc = False
    req.segmentation2.directory = d2
    req.segmentation2.split_cc = False
    req.segmentation2.min_size = 0
    if not np.isnan(float(g['threshold_%d' % i])):
      req.segmentation1.threshold = float(g['threshold_%d' % i])
    if str(g['mask_%d' % i]):
      req.segmentation1.mask.masks.add().coordinate_expression.expression = str(g['mask_%d' % i])
    origins = {int(k): ((tuple(int(v) for v in s)), int(it), float(w)) for k, s, it, w in zip(
        g['origin_ids_%d' % i], g['origin_start_%d' % i], g['origin_iters_%d' % i], g['origin_wall_%d' % i])}
    out.append(dict(tag=str(g['ctag_%d' % i]), request=req, corner=corner, loaded1=g['loaded1_%d' % i],
                    loaded2=g['loaded2_%d' % i], loaded1_origin_ids=[int(k) for k in g['loaded1_origin_ids_%d' % i]],
                    seg=g['seg_%d' % i], origins=origins, stale=[int(k) for k in g['stale_%d' % i]]))
  return out


def plain_origins(origins):
  return {int(k): (tuple(int(v) for v in o.start_zyx), int(o.iters), float(o.walltime_sec)) for k, o in origins.items()}


def test_fixture_covers_the_cases():
  cases = {c[0]: c for c in split_cases()}
  assert {str(cases['reduce_%s' % t][5].dtype) for t in ('u8', 'u16', 'u32', 'u64')} == {
      'uint8', 'uint16', 'uint32', 'uint64'}
  assert cases['a_ge_2_63_no_0'][1].min() > 0 and cases['a_ge_2_63_no_0'][1].max() >= 2**63
  assert cases['a_ge_2_32_with_0'][1].min() == 0 and cases['a_ge_2_32_with_0'][1].max() >= 2**32
  assert cases['b_ge_2_32'][2].max() >= 2**32
  # ties: the smallest b wins among equal counts
  ties = cases['ties']
  assert ties[5][0, 0, 3] == 5 and ties[5][0, 2, 4] == 8
  # (a, 0) pairs survive, (0, b) pairs never do
  _, a, b, _, _, out, _, _ = cases['zero_pairs']
  assert (out[(b == 0) & (a > 0)] > 0).any() and not out[a == 0].any()
  assert {c[7] for c in cases.values()} == {'', 'ValueError', 'TypeError'}
  for c in consensus_cases_from_fixture():
    assert c['stale'] and set(c['stale']) <= set(c['origins'])


def consensus_cases_from_fixture():
  g = np.load(GOLDEN)
  return [dict(stale=[int(k) for k in g['stale_%d' % i]], origins=[int(k) for k in g['origin_ids_%d' % i]])
          for i in range(int(g['n_consensus']))]


@pytest.mark.parametrize('case', split_cases(), ids=lambda c: c[0])
def test_oracle_equals_reference(case):
  tag, a, b, min_size, ctype, want, after, error = case
  v1, b_in = a.copy(), b.copy()
  if error:
    with pytest.raises(ERRORS[error]):
      oc.compute_consensus_for_segmentations(v1, b, min_size, ctype)
    return
  got = oc.compute_consensus_for_segmentations(v1, b, min_size, ctype)
  assert got.dtype == want.dtype and np.array_equal(got, want), tag
  assert np.array_equal(v1, after) and np.array_equal(b, b_in), tag


def test_oracle_equals_reference_compute_consensus(tmp_path):
  for c in consensus_cases(tmp_path):
    v1, o1 = storage.load_segmentation_from_source(c['request'].segmentation1, c['corner'])
    v2, _ = storage.load_segmentation_from_source(c['request'].segmentation2, c['corner'])
    seg = oc.compute_consensus_for_segmentations(v1, v2, c['request'].split_min_size)
    assert seg.dtype == c['seg'].dtype and np.array_equal(seg, c['seg']), c['tag']
    assert plain_origins(oc.relabeled_origins(seg, o1)) == c['origins'], c['tag']


def test_load_segmentation_from_source_equals_reference(tmp_path):
  for c in consensus_cases(tmp_path):
    for k, want in ((1, c['loaded1']), (2, c['loaded2'])):
      got, origins = storage.load_segmentation_from_source(getattr(c['request'], 'segmentation%d' % k), c['corner'])
      assert got.dtype == np.uint64 and np.array_equal(got, want), (c['tag'], k)
      if k == 1:
        assert sorted(int(x) for x in origins) == c['loaded1_origin_ids'], c['tag']


def test_load_segmentation_from_source_rejects_connected_components(tmp_path):
  d1, _, corner = write_sources(tmp_path)
  src = consensus_pb2.ConsensusRequest().segmentation1
  src.directory = d1
  with pytest.raises(NotImplementedError, match='split_cc'):
    storage.load_segmentation_from_source(src, corner)        # unset: the reference's default is True
  src.split_cc = True
  with pytest.raises(NotImplementedError, match='split_cc'):
    storage.load_segmentation_from_source(src, corner)
  src.split_cc = False
  src.min_size = 3
  with pytest.raises(NotImplementedError, match='min_size'):
    storage.load_segmentation_from_source(src, corner)
  src.min_size = 0
  seg, _ = storage.load_segmentation_from_source(src, corner)
  assert seg.dtype == np.uint64 and seg.any()


def test_load_segmentation_from_source_all_zero(tmp_path):
  """An all-zero file comes back without origins, as the reference's load_segmentation returns it."""
  corner = (0, 0, 0)
  d = str(tmp_path / 'empty')
  storage.save_subvolume(np.zeros((3, 4, 5), np.uint64), {1: storage.OriginInfo((0, 0, 0), 1, 0.0)},
                         storage.segmentation_path(d, corner))
  src = consensus_pb2.ConsensusRequest().segmentation1
  src.directory = d
  src.split_cc = False
  seg, origins = storage.load_segmentation_from_source(src, corner)
  assert seg.dtype == np.uint64 and seg.shape == (3, 4, 5) and not seg.any() and origins == {}


# consensus.proto:22-36 — (field, number, type, message or enum type)
PROTO = [('segmentation1', 1, 'message', 'ffn.SegmentationSource'),
         ('segmentation2', 2, 'message', 'ffn.SegmentationSource'),
         ('segmentation_output_dir', 3, 'string', None),
         ('type', 4, 'enum', 'ffn.ConsensusRequest.ConsensusType'),
         ('split_min_size', 7, 'int32', None)]


def test_consensus_request_matches_consensus_proto():
  from google.protobuf import descriptor as d
  types = {d.FieldDescriptor.TYPE_INT32: 'int32', d.FieldDescriptor.TYPE_STRING: 'string',
           d.FieldDescriptor.TYPE_MESSAGE: 'message', d.FieldDescriptor.TYPE_ENUM: 'enum'}
  desc = consensus_pb2.ConsensusRequest.DESCRIPTOR
  assert desc.full_name == 'ffn.ConsensusRequest'
  assert desc.file.name == 'inference/consensus.proto' and desc.file.package == 'ffn'
  assert len(desc.fields) == len(PROTO)
  for name, number, ftype, tname in PROTO:
    f = desc.fields_by_name[name]
    assert (f.number, types[f.type]) == (number, ftype), name
    assert not f.is_repeated, name
    sub = f.message_type or f.enum_type
    assert (sub.full_name if sub else None) == tname, name
  enum = desc.enum_types_by_name['ConsensusType']
  assert [(v.name, v.number) for v in enum.values] == [('CONSENSUS_SPLIT', 2)]
  req = consensus_pb2.ConsensusRequest()
  assert req.type == req.CONSENSUS_SPLIT == 2   # the first (only) value is the proto2 default
  req.segmentation1.threshold = 0.5
  back = consensus_pb2.ConsensusRequest.FromString(req.SerializeToString())
  assert back.segmentation1.HasField('threshold') and not back.segmentation1.HasField('split_cc')


def test_ffn_namespace_aliases():
  from ffn.inference import consensus, consensus_pb2 as pb2
  from ffn_b200.inference import consensus as impl
  assert consensus is impl and pb2 is consensus_pb2
  for name in ('compute_consensus_for_segmentations', 'compute_consensus'):
    assert callable(getattr(consensus, name)), name


@pytest.mark.parametrize('case', [c for c in split_cases() if c[7]], ids=lambda c: c[0])
def test_input_errors_decided_on_the_host(case):
  """Shape, dtype and consensus-type errors raise what the reference raises, before any device work."""
  from ffn_b200.inference import consensus
  tag, a, b, min_size, ctype, _, _, error = case
  req = consensus_pb2.ConsensusRequest(split_min_size=min_size)
  if ctype != 2:
    class Req:
      type = ctype
      split_min_size = min_size
    req = Req()
  with pytest.raises(ERRORS[error]):
    consensus.compute_consensus_for_segmentations(a.copy(), b, req)
  with pytest.raises(ValueError):
    segmentation.split_segmentation_by_intersection(np.zeros(0, np.uint64), np.zeros(0, np.uint64), 0)
