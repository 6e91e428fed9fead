"""Wire-compatible protocol buffers for the inference request, built at import time.

The reference ships pre-3.20 generated `*_pb2.py` files (ffn/inference/inference_pb2.py,
ffn/utils/{bounding_box,vector}_pb2.py) that no longer import under current protobuf runtimes,
and `protoc` is not available.  The messages are therefore declared here programmatically with
the SAME package names, message names, field names, numbers, types, labels and defaults as
ffn/inference/inference.proto:22-330, ffn/utils/bounding_box.proto:26-48 and
ffn/utils/vector.proto — so text-format requests (configs/*.pbtxt) and serialized requests
embedded in result files parse unchanged.
"""

from google.protobuf import descriptor_pb2
from google.protobuf import descriptor_pool
from google.protobuf import message_factory

_F = descriptor_pb2.FieldDescriptorProto
_T = {
    'double': _F.TYPE_DOUBLE, 'float': _F.TYPE_FLOAT, 'int64': _F.TYPE_INT64,
    'uint64': _F.TYPE_UINT64, 'int32': _F.TYPE_INT32, 'bool': _F.TYPE_BOOL,
    'string': _F.TYPE_STRING,
}


def _field(msg, name, number, ftype, repeated=False, default=None, oneof=None):
  f = msg.field.add()
  f.name = name
  f.number = number
  f.label = _F.LABEL_REPEATED if repeated else _F.LABEL_OPTIONAL
  if ftype in _T:
    f.type = _T[ftype]
  elif ftype.startswith('enum:'):
    f.type = _F.TYPE_ENUM
    f.type_name = ftype[5:]
  else:
    f.type = _F.TYPE_MESSAGE
    f.type_name = ftype
  if default is not None:
    f.default_value = default
  if oneof is not None:
    f.oneof_index = oneof
  return f


def _vector_file():
  fd = descriptor_pb2.FileDescriptorProto()
  fd.name = 'utils/vector.proto'
  fd.package = 'ffn.proto'
  fd.syntax = 'proto2'
  for name, comps, t in (('Vector2d', 'xy', 'double'), ('Vector2i', 'xy', 'int32'),
                         ('Vector3d', 'xyz', 'double'), ('Vector3f', 'xyz', 'float'),
                         ('Vector3j', 'xyz', 'int64')):
    m = fd.message_type.add()
    m.name = name
    for i, c in enumerate(comps):
      _field(m, c, i + 1, t)
  for name in ('Vector2d', 'Vector2i', 'Vector3d', 'Vector3f', 'Vector3j'):
    m = fd.message_type.add()
    m.name = name + 'List'
    _field(m, 'vectors', 1, '.ffn.proto.' + name, repeated=True)
  return fd


def _bounding_box_file():
  fd = descriptor_pb2.FileDescriptorProto()
  fd.name = 'utils/bounding_box.proto'
  fd.package = 'ffn'
  fd.syntax = 'proto2'
  fd.dependency.append('utils/vector.proto')
  m = fd.message_type.add()
  m.name = 'BoundingBox'
  _field(m, 'start', 1, '.ffn.proto.Vector3j')
  _field(m, 'size', 2, '.ffn.proto.Vector3j')
  _field(m, 'description', 3, 'string')
  _field(m, 'object_label', 4, 'uint64')
  m = fd.message_type.add()
  m.name = 'BoundingBoxes'
  _field(m, 'box', 1, '.ffn.BoundingBox', repeated=True)
  return fd


def _inference_file():
  fd = descriptor_pb2.FileDescriptorProto()
  fd.name = 'inference/inference.proto'
  fd.package = 'ffn'
  fd.syntax = 'proto2'
  fd.dependency.extend(['utils/vector.proto', 'utils/bounding_box.proto'])

  m = fd.message_type.add()
  m.name = 'DecoratedVolume'
  m.oneof_decl.add().name = 'volume_path'
  _field(m, 'volinfo', 1, 'string', oneof=0)
  _field(m, 'hdf5', 3, 'string', oneof=0)
  _field(m, 'tensorstore', 4, 'string', oneof=0)
  _field(m, 'decorator_specs', 2, 'string')

  m = fd.message_type.add()
  m.name = 'MaskChannelConfig'
  _field(m, 'channel', 1, 'int32')
  _field(m, 'min_value', 2, 'float')
  _field(m, 'max_value', 3, 'float')
  _field(m, 'values', 5, 'uint64', repeated=True)
  _field(m, 'invert', 4, 'bool')

  m = fd.message_type.add()
  m.name = 'ImageMaskOptions'
  _field(m, 'channels', 1, '.ffn.MaskChannelConfig', repeated=True)

  m = fd.message_type.add()
  m.name = 'VolumeMaskOptions'
  _field(m, 'mask', 1, '.ffn.DecoratedVolume')
  _field(m, 'channels', 2, '.ffn.MaskChannelConfig', repeated=True)

  m = fd.message_type.add()
  m.name = 'CoordinateExpressionOptions'
  _field(m, 'expression', 1, 'string')

  m = fd.message_type.add()
  m.name = 'MaskConfig'
  m.oneof_decl.add().name = 'source'
  _field(m, 'volume', 1, '.ffn.VolumeMaskOptions', oneof=0)
  _field(m, 'image', 2, '.ffn.ImageMaskOptions', oneof=0)
  _field(m, 'coordinate_expression', 3, '.ffn.CoordinateExpressionOptions', oneof=0)
  _field(m, 'invert', 4, 'bool')

  m = fd.message_type.add()
  m.name = 'MaskConfigs'
  _field(m, 'masks', 1, '.ffn.MaskConfig', repeated=True)

  m = fd.message_type.add()
  m.name = 'SegmentationSource'
  _field(m, 'directory', 1, 'string')
  _field(m, 'threshold', 2, 'float')
  _field(m, 'split_cc', 3, 'bool')
  _field(m, 'min_size', 4, 'int32')
  _field(m, 'mask', 5, '.ffn.MaskConfigs')

  m = fd.message_type.add()
  m.name = 'InferenceOptions'
  _field(m, 'init_activation', 1, 'float')
  _field(m, 'pad_value', 2, 'float')
  _field(m, 'move_threshold', 3, 'float')
  _field(m, 'disco_seed_threshold', 5, 'float')
  _field(m, 'min_boundary_dist', 6, '.ffn.proto.Vector3j')
  _field(m, 'segment_threshold', 7, 'float')
  _field(m, 'min_segment_size', 8, 'int32')
  r = m.reserved_range.add()
  r.start, r.end = 4, 5
  m.reserved_name.append('consistency_threshold')

  m = fd.message_type.add()
  m.name = 'AlignmentOptions'
  e = m.enum_type.add()
  e.name = 'AlignType'
  for n, v in (('UNKNOWN_ALIGNMENT', 0), ('NO_ALIGNMENT', 1)):
    ev = e.value.add()
    ev.name, ev.number = n, v
  _field(m, 'type', 1, 'enum:.ffn.AlignmentOptions.AlignType', default='NO_ALIGNMENT')
  _field(m, 'save_raw', 6, 'bool')

  m = fd.message_type.add()
  m.name = 'InferenceRequest'
  _field(m, 'image', 24, '.ffn.DecoratedVolume')
  _field(m, 'image_mean', 2, 'float')
  _field(m, 'image_stddev', 3, 'float')
  _field(m, 'reference_histogram', 4, 'string')
  _field(m, 'histogram_masks', 26, '.ffn.MaskConfig', repeated=True)
  _field(m, 'masks', 5, '.ffn.MaskConfig', repeated=True)
  _field(m, 'seed_masks', 30, '.ffn.MaskConfig', repeated=True)
  _field(m, 'shift_mask', 6, '.ffn.DecoratedVolume')
  _field(m, 'shift_mask_fov', 22, '.ffn.BoundingBox')
  _field(m, 'shift_mask_scale', 7, 'int32')
  _field(m, 'shift_mask_threshold', 8, 'int32')
  _field(m, 'movement_policy_name', 9, 'string')
  _field(m, 'movement_policy_args', 10, 'string')
  _field(m, 'model_name', 11, 'string')
  _field(m, 'model_args', 12, 'string')
  _field(m, 'model_checkpoint_path', 13, 'string')
  _field(m, 'batch_size', 27, 'int32', default='1')
  _field(m, 'concurrent_requests', 28, 'int32', default='1')
  _field(m, 'inference_options', 14, '.ffn.InferenceOptions')
  _field(m, 'segmentation_output_dir', 15, 'string')
  _field(m, 'checkpoint_interval', 16, 'int32')
  _field(m, 'seed_policy', 17, 'string')
  _field(m, 'seed_policy_args', 19, 'string')
  _field(m, 'alignment_options', 20, '.ffn.AlignmentOptions')
  _field(m, 'init_segmentation', 25, '.ffn.DecoratedVolume')
  r = m.reserved_range.add()
  r.start, r.end = 18, 19
  m.reserved_name.append('self_prediction')

  m = fd.message_type.add()
  m.name = 'ResegmentationPoint'
  _field(m, 'id_a', 1, 'uint64')
  _field(m, 'id_b', 2, 'uint64')
  _field(m, 'point', 3, '.ffn.proto.Vector3j')

  m = fd.message_type.add()
  m.name = 'ResegmentationRequest'
  _field(m, 'inference', 1, '.ffn.InferenceRequest')
  _field(m, 'points', 2, '.ffn.ResegmentationPoint', repeated=True)
  _field(m, 'radius', 5, '.ffn.proto.Vector3j')
  _field(m, 'output_directory', 6, 'string')
  _field(m, 'subdir_digits', 7, 'int32')
  _field(m, 'max_retry_iters', 8, 'int32', default='1')
  _field(m, 'exclusion_radius', 9, '.ffn.proto.Vector3j')
  _field(m, 'init_exclusion_radius', 11, '.ffn.proto.Vector3j')
  _field(m, 'segment_recovery_fraction', 10, 'float')
  _field(m, 'terminate_early', 12, 'bool')
  _field(m, 'analysis_radius', 13, '.ffn.proto.Vector3j')

  m = fd.message_type.add()
  m.name = 'CounterValue'
  _field(m, 'name', 1, 'string')
  _field(m, 'value', 2, 'int64')

  m = fd.message_type.add()
  m.name = 'TaskCounters'
  _field(m, 'counters', 1, '.ffn.CounterValue', repeated=True)
  _field(m, 'point', 2, '.ffn.proto.Vector3j')
  _field(m, 'filename', 3, 'string')
  return fd


def _resegmentation_file():
  """ffn/inference/resegmentation.proto:22-113: statistics of resegmentation results."""
  fd = descriptor_pb2.FileDescriptorProto()
  fd.name = 'inference/resegmentation.proto'
  fd.package = 'ffn'
  fd.syntax = 'proto2'
  fd.dependency.append('utils/vector.proto')

  m = fd.message_type.add()
  m.name = 'EndpointResegmentationResult'
  o = m.nested_type.add()
  o.name = 'OverlapInfo'
  _field(o, 'num_overlapping', 1, 'int32')
  _field(o, 'num_original', 2, 'int32')
  e = m.nested_type.add()   # what protoc generates for map<uint64, OverlapInfo>
  e.name = 'OverlapsEntry'
  e.options.map_entry = True
  _field(e, 'key', 1, 'uint64')
  _field(e, 'value', 2, '.ffn.EndpointResegmentationResult.OverlapInfo')
  _field(m, 'id', 1, 'uint64')
  _field(m, 'start', 2, '.ffn.proto.Vector3j')
  _field(m, 'num_voxels', 3, 'int32')
  _field(m, 'overlaps', 4, '.ffn.EndpointResegmentationResult.OverlapsEntry', repeated=True)
  _field(m, 'source', 5, '.ffn.EndpointResegmentationResult.OverlapInfo')
  _field(m, 'segmentation_radius', 6, '.ffn.proto.Vector3j')
  _field(m, 'tag', 7, 'string')

  m = fd.message_type.add()
  m.name = 'PairResegmentationResult'
  s = m.nested_type.add()
  s.name = 'SegmentResult'
  _field(s, 'origin', 1, '.ffn.proto.Vector3j')
  _field(s, 'num_voxels', 2, 'int32')
  _field(s, 'deleted_voxels', 3, 'int32')
  _field(s, 'segment_a_consistency', 4, 'float')
  _field(s, 'segment_b_consistency', 5, 'float')
  _field(s, 'max_edt', 6, 'float')
  r = m.nested_type.add()
  r.name = 'EvalResult'
  _field(r, 'radius', 1, '.ffn.proto.Vector3j')
  _field(r, 'iou', 2, 'float')
  _field(r, 'from_a', 3, '.ffn.PairResegmentationResult.SegmentResult')
  _field(r, 'from_b', 4, '.ffn.PairResegmentationResult.SegmentResult')
  _field(r, 'max_edt_a', 5, 'float')
  _field(r, 'max_edt_b', 6, 'float')
  _field(r, 'num_voxels_a', 7, 'int32')
  _field(r, 'num_voxels_b', 8, 'int32')
  _field(m, 'point', 1, '.ffn.proto.Vector3j')
  _field(m, 'id_a', 2, 'uint64')
  _field(m, 'id_b', 3, 'uint64')
  _field(m, 'segmentation_radius', 4, '.ffn.proto.Vector3j')
  _field(m, 'tag', 5, 'string')
  _field(m, 'eval', 6, '.ffn.PairResegmentationResult.EvalResult')
  return fd


def _consensus_file():
  """ffn/inference/consensus.proto:22-36: the request of split consensus."""
  fd = descriptor_pb2.FileDescriptorProto()
  fd.name = 'inference/consensus.proto'
  fd.package = 'ffn'
  fd.syntax = 'proto2'
  fd.dependency.extend(['utils/vector.proto', 'inference/inference.proto'])

  m = fd.message_type.add()
  m.name = 'ConsensusRequest'
  e = m.enum_type.add()
  e.name = 'ConsensusType'
  ev = e.value.add()
  ev.name, ev.number = 'CONSENSUS_SPLIT', 2
  _field(m, 'segmentation1', 1, '.ffn.SegmentationSource')
  _field(m, 'segmentation2', 2, '.ffn.SegmentationSource')
  _field(m, 'segmentation_output_dir', 3, 'string')
  _field(m, 'type', 4, 'enum:.ffn.ConsensusRequest.ConsensusType')
  _field(m, 'split_min_size', 7, 'int32')
  return fd


def _build():
  pool = descriptor_pool.DescriptorPool()   # private pool: never clashes with a real ffn install
  classes = {}
  for fd in (_vector_file(), _bounding_box_file(), _inference_file(), _resegmentation_file(), _consensus_file()):
    pool.Add(fd)
    file_desc = pool.FindFileByName(fd.name)
    for name, desc in file_desc.message_types_by_name.items():
      classes[desc.full_name] = message_factory.GetMessageClass(desc)
  return pool, classes


_POOL, _CLASSES = _build()

Vector3j = _CLASSES['ffn.proto.Vector3j']
Vector3d = _CLASSES['ffn.proto.Vector3d']
Vector3f = _CLASSES['ffn.proto.Vector3f']
BoundingBox = _CLASSES['ffn.BoundingBox']
BoundingBoxes = _CLASSES['ffn.BoundingBoxes']
DecoratedVolume = _CLASSES['ffn.DecoratedVolume']
MaskChannelConfig = _CLASSES['ffn.MaskChannelConfig']
ImageMaskOptions = _CLASSES['ffn.ImageMaskOptions']
VolumeMaskOptions = _CLASSES['ffn.VolumeMaskOptions']
CoordinateExpressionOptions = _CLASSES['ffn.CoordinateExpressionOptions']
MaskConfig = _CLASSES['ffn.MaskConfig']
MaskConfigs = _CLASSES['ffn.MaskConfigs']
SegmentationSource = _CLASSES['ffn.SegmentationSource']
InferenceOptions = _CLASSES['ffn.InferenceOptions']
AlignmentOptions = _CLASSES['ffn.AlignmentOptions']
InferenceRequest = _CLASSES['ffn.InferenceRequest']
ResegmentationPoint = _CLASSES['ffn.ResegmentationPoint']
ResegmentationRequest = _CLASSES['ffn.ResegmentationRequest']
CounterValue = _CLASSES['ffn.CounterValue']
TaskCounters = _CLASSES['ffn.TaskCounters']
EndpointResegmentationResult = _CLASSES['ffn.EndpointResegmentationResult']
PairResegmentationResult = _CLASSES['ffn.PairResegmentationResult']
ConsensusRequest = _CLASSES['ffn.ConsensusRequest']
