"""Resegmentation analysis on the host: the oracle against the fixture written by the reference's own module
(tests/golden/make_golden_reseg_analysis.py), the result messages against resegmentation.proto, file-name parsing
and the error paths that are decided before any device work."""
import os

import numpy as np
import pytest

from ffn_b200.inference import resegmentation_analysis as ra
from ffn_b200.inference import resegmentation_pb2
from oracle import reseg_analysis as ora

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reseg_analysis_ref.npz')


def fixture_cases(tmp_path):
  """(tag, kind, path, volume, radius, analysis, voxel, threshold, expected bytes, expected error name) per case."""
  g = np.load(GOLDEN)
  out = []
  for i in range(int(g['n'])):
    path = tmp_path / ('%02d' % i) / str(g['name_%d' % i])
    path.parent.mkdir()
    path.write_bytes(g['file_%d' % i].tobytes())
    out.append((str(g['tag_%d' % i]), str(g['kind_%d' % i]), str(path), g['volume_%d' % int(g['volume_%d_of' % i])],
                tuple(int(v) for v in g['radius_%d' % i]), tuple(int(v) for v in g['analysis_%d' % i]),
                tuple(int(v) for v in g['voxel_%d' % i]), float(g['threshold_%d' % i]), g['expect_%d' % i].tobytes(),
                str(g['error_%d' % i])))
  return out


def test_oracle_reproduces_reference_fixture(tmp_path):
  cases = fixture_cases(tmp_path)
  assert {c[1] for c in cases} == {'pair', 'endpoint'} and len(cases) == 12
  for tag, kind, path, vol, radius, analysis, voxel, threshold, expect, error in cases:
    if kind == 'pair':
      call = lambda: ora.evaluate_pair_resegmentation(path, vol, radius, analysis, voxel, threshold)  # noqa: E731
    else:
      call = lambda: ora.evaluate_endpoint_resegmentation(path, vol, radius, threshold)  # noqa: E731
    if error:
      with pytest.raises(getattr(ora, error)):
        call()
      continue
    got = call()
    assert got.SerializeToString(deterministic=True) == expect, tag
    want = type(got).FromString(expect)
    assert got == want, tag


def test_fixture_pins_a_mask_without_background(tmp_path):
  """In `pair_big_ids_full` the first resegmented object fills the whole analysis box, so its distance transform has
  no background voxel.  The reference's value there is scipy's: (Z wz)^2 + ((Y-1) wy)^2 + ((X-1) wx)^2."""
  from ffn_b200.inference import storage
  case = {c[0]: c for c in fixture_cases(tmp_path)}['pair_big_ids_full']
  _, _, path, _, radius, analysis, voxel, threshold, expect, _ = case
  probs = np.load(path, allow_pickle=True)['probs']
  delta = np.array(radius) - np.array(analysis)
  box = tuple(slice(d, d + 2 * a + 1) for d, a in zip(delta, analysis))
  assert (np.nan_to_num(storage.dequantize_probability(probs[0][box])) >= threshold).all()
  want = resegmentation_pb2.PairResegmentationResult.FromString(expect)
  shape = [2 * a + 1 for a in analysis]
  d2 = (shape[0] * voxel[0]) ** 2 + ((shape[1] - 1) * voxel[1]) ** 2 + ((shape[2] - 1) * voxel[2]) ** 2
  assert want.eval.from_a.num_voxels == np.prod(shape)
  assert want.eval.from_a.max_edt == float(np.float32(np.sqrt(float(d2))))


# resegmentation.proto:22-113 — (field, number, type, label, message type) per message
_F = 'optional'
PROTO = {
    'ffn.EndpointResegmentationResult': [
        ('id', 1, 'uint64', _F, None), ('start', 2, 'message', _F, 'ffn.proto.Vector3j'),
        ('num_voxels', 3, 'int32', _F, None),
        ('overlaps', 4, 'message', 'repeated', 'ffn.EndpointResegmentationResult.OverlapsEntry'),
        ('source', 5, 'message', _F, 'ffn.EndpointResegmentationResult.OverlapInfo'),
        ('segmentation_radius', 6, 'message', _F, 'ffn.proto.Vector3j'), ('tag', 7, 'string', _F, None)],
    'ffn.EndpointResegmentationResult.OverlapInfo': [
        ('num_overlapping', 1, 'int32', _F, None), ('num_original', 2, 'int32', _F, None)],
    'ffn.PairResegmentationResult': [
        ('point', 1, 'message', _F, 'ffn.proto.Vector3j'), ('id_a', 2, 'uint64', _F, None),
        ('id_b', 3, 'uint64', _F, None), ('segmentation_radius', 4, 'message', _F, 'ffn.proto.Vector3j'),
        ('tag', 5, 'string', _F, None), ('eval', 6, 'message', _F, 'ffn.PairResegmentationResult.EvalResult')],
    'ffn.PairResegmentationResult.SegmentResult': [
        ('origin', 1, 'message', _F, 'ffn.proto.Vector3j'), ('num_voxels', 2, 'int32', _F, None),
        ('deleted_voxels', 3, 'int32', _F, None), ('segment_a_consistency', 4, 'float', _F, None),
        ('segment_b_consistency', 5, 'float', _F, None), ('max_edt', 6, 'float', _F, None)],
    'ffn.PairResegmentationResult.EvalResult': [
        ('radius', 1, 'message', _F, 'ffn.proto.Vector3j'), ('iou', 2, 'float', _F, None),
        ('from_a', 3, 'message', _F, 'ffn.PairResegmentationResult.SegmentResult'),
        ('from_b', 4, 'message', _F, 'ffn.PairResegmentationResult.SegmentResult'),
        ('max_edt_a', 5, 'float', _F, None), ('max_edt_b', 6, 'float', _F, None),
        ('num_voxels_a', 7, 'int32', _F, None), ('num_voxels_b', 8, 'int32', _F, None)],
}


def test_result_messages_match_resegmentation_proto():
  from google.protobuf import descriptor as d
  types = {d.FieldDescriptor.TYPE_UINT64: 'uint64', d.FieldDescriptor.TYPE_INT32: 'int32',
           d.FieldDescriptor.TYPE_FLOAT: 'float', d.FieldDescriptor.TYPE_STRING: 'string',
           d.FieldDescriptor.TYPE_MESSAGE: 'message'}
  pool = resegmentation_pb2.PairResegmentationResult.DESCRIPTOR.file.pool
  for full, fields in PROTO.items():
    desc = pool.FindMessageTypeByName(full)
    assert desc.file.name == 'inference/resegmentation.proto' and desc.file.package == 'ffn'
    assert len(desc.fields) == len(fields), full
    for name, number, ftype, label, mtype in fields:
      f = desc.fields_by_name[name]
      assert (f.number, types[f.type]) == (number, ftype), (full, name)
      assert f.is_repeated == (label == 'repeated'), (full, name)
      assert (f.message_type.full_name if f.message_type else None) == mtype, (full, name)
  entry = pool.FindMessageTypeByName('ffn.EndpointResegmentationResult.OverlapsEntry')
  assert entry.GetOptions().map_entry
  assert [(f.name, f.number, types[f.type]) for f in entry.fields] == [('key', 1, 'uint64'), ('value', 2, 'message')]
  # map semantics, and the reference module's spelling of the endpoint message
  m = resegmentation_pb2.EndpointSegmentationResult()
  assert resegmentation_pb2.EndpointSegmentationResult is resegmentation_pb2.EndpointResegmentationResult
  m.overlaps[2**64 - 1].num_overlapping = 3
  m.overlaps[0].num_original = 5
  back = resegmentation_pb2.EndpointResegmentationResult.FromString(m.SerializeToString(deterministic=True))
  assert dict((k, (v.num_overlapping, v.num_original)) for k, v in back.overlaps.items()) == {
      2**64 - 1: (3, 0), 0: (0, 5)}


def test_ffn_namespace_aliases():
  from ffn.inference import resegmentation_analysis, resegmentation_pb2 as pb2
  assert resegmentation_analysis is ra and pb2 is resegmentation_pb2
  for name in ('InvalidBaseSegmentatonError', 'IncompleteResegmentationError', 'compute_iou',
               'evaluate_segmentation_result', 'parse_resegmentation_filename', 'evaluate_endpoint_resegmentation',
               'evaluate_pair_resegmentation', 'evaluate_pair_resegmentations', 'evaluate_endpoint_resegmentations'):
    assert callable(getattr(ra, name)), name


def test_parse_filename_and_iou():
  assert ra.parse_resegmentation_filename('/a/b/9223372036854788153-12_at_30_36_7.npz') == (
      9223372036854788153, 12, 30, 36, 7)
  assert ra.parse_resegmentation_filename('3-0_at_1_2_3.npz') == (3, 0, 1, 2, 3)
  with pytest.raises(AttributeError):
    ra.parse_resegmentation_filename('no-match.npz')
  reseg = np.zeros((2, 2, 3, 4), bool)
  reseg[0, 0] = True
  reseg[1, :, 0] = True
  assert ra.compute_iou(reseg) == 4 / 16.0


def test_errors_decided_on_the_host(tmp_path):
  """A file with one object is incomplete, before any device work; a batch carries the error in its slot.  Bad voxel
  sizes and boxes that do not match the probability maps are rejected."""
  cases = {c[0]: c for c in fixture_cases(tmp_path)}
  _, _, path, vol, radius, analysis, voxel, _, _, _ = cases['pair_incomplete']
  with pytest.raises(ra.IncompleteResegmentationError):
    ra.evaluate_pair_resegmentation(path, vol, radius, analysis, voxel)
  out = ra.evaluate_pair_resegmentations([path, path], vol, radius, analysis, voxel)
  assert len(out) == 2 and all(isinstance(e, ra.IncompleteResegmentationError) for e in out)
  _, _, good, vol, radius, analysis, voxel, _, _, _ = cases['pair_merge']
  for bad in ((30, 8, 8.5), (0, 8, 8), (8, 8)):
    with pytest.raises(ValueError):
      ra.evaluate_pair_resegmentations([good], vol, radius, analysis, bad)
  with pytest.raises(ValueError):   # the analysis box must lie inside the resegmentation box
    ra.evaluate_pair_resegmentations([good], vol, radius, tuple(r + 1 for r in radius), voxel)
  _, _, ep, vol, radius, _, _, _, _, _ = cases['endpoint_spill']
  with pytest.raises(ValueError):   # the segmentation box must match the probability map
    ra.evaluate_endpoint_resegmentations([ep], vol, tuple(r - 1 for r in radius))
  with pytest.raises(ValueError):   # negative ids cannot be overlap keys
    ra.evaluate_endpoint_resegmentations([ep], vol.astype(np.int64) - 1, radius)
