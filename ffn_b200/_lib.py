"""ctypes binding of libffn_b200.so (the C ABI in include/ffn_b200.h).

The library is built in-tree by ``ffn_b200/build.py``.  There is deliberately no fallback: if the
shared object is missing or cannot be loaded, importing the engine raises.
"""

from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, 'libffn_b200.so')

COMPUTE_FP16_TC = 0
COMPUTE_FP32 = 1
COMPUTE_FP16X2_TC = 2   # fp16 hi+lo split operands on the tensor cores: near-fp32, label-exact parity mode
IMAGE_U8 = 0
IMAGE_F32 = 1
ARRAY_SEED = 0
ARRAY_SEGMENTATION = 1
ARRAY_QPROB = 2
ARRAY_IMAGE = 3
MASK_MOVEMENT = 0
MASK_SEED = 1
SEED_POLICY_KINDS = {'peaks_2d': 0, 'fill_empty': 1, 'max_peaks': 2}   # FFN_SEED_*
OPTIMIZERS = {'sgd': 0, 'momentum': 1, 'adam': 2}   # FFN_OPT_*

EXPORTS = [
    'ffn_last_error', 'ffn_engine_create', 'ffn_engine_destroy', 'ffn_engine_set_compute_mode', 'ffn_engine_set_chains', 'ffn_engine_set_grid',
    'ffn_engine_set_step_chunk', 'ffn_engine_info', 'ffn_engine_profile', 'ffn_engine_trace', 'ffn_face_table', 'ffn_predict', 'ffn_canvas_create', 'ffn_canvas_destroy',
    'ffn_canvas_set_mask', 'ffn_canvas_segment_at', 'ffn_canvas_segment_all',
    'ffn_canvas_update_at', 'ffn_canvas_init_seed', 'ffn_canvas_read', 'ffn_canvas_write',
    'ffn_canvas_policy_state_size', 'ffn_canvas_policy_state_get', 'ffn_canvas_policy_state_set',
    'ffn_canvas_set_resume', 'ffn_canvas_trace', 'ffn_canvas_seed_peaks', 'ffn_canvas_seed_policy', 'ffn_canvas_set_max_id', 'ffn_canvas_get_counters', 'ffn_canvas_spec_stats', 'ffn_canvas_sched_stats', 'ffn_canvas_device_ptr',
    'ffn_canvas_add_id_offset', 'ffn_decision_points', 'ffn_reseg_eval', 'ffn_split_intersection', 'ffn_compute_partitions',
    'ffn_partition_rows', 'ffn_coordinate_records', 'ffn_clean_up', 'ffn_trainer_create', 'ffn_trainer_destroy',
    'ffn_trainer_step', 'ffn_trainer_gradients', 'ffn_trainer_get_weights', 'ffn_trainer_train', 'ffn_examples_create',
    'ffn_examples_destroy', 'ffn_examples_next', 'ffn_examples_update', 'ffn_examples_read_seeds', 'ffn_examples_tracker',
    'ffn_selftest_wgmma',
]


class ModelDesc(C.Structure):
  _fields_ = [('fov_zyx', C.c_int32 * 3), ('deltas_zyx', C.c_int32 * 3), ('depth', C.c_int32),
              ('features', C.c_int32)]


class Options(C.Structure):
  _fields_ = [('init_activation', C.c_float), ('pad_value', C.c_float),
              ('move_threshold', C.c_float), ('segment_threshold', C.c_float),
              ('disco_seed_threshold', C.c_float), ('policy_score_threshold', C.c_double),
              ('min_boundary_dist_zyx', C.c_int32 * 3), ('min_segment_size', C.c_int32)]


class SegStats(C.Structure):
  _fields_ = [('iters', C.c_int64), ('min_pos', C.c_int32 * 3), ('max_pos', C.c_int32 * 3),
              ('seed_got_too_weak', C.c_int32), ('queue_len', C.c_int32), ('finished', C.c_int32),
              ('reserved', C.c_int32)]


class Origin(C.Structure):
  _fields_ = [('id', C.c_int32), ('start_zyx', C.c_int32 * 3), ('iters', C.c_int64),
              ('walltime_sec', C.c_double)]


class Overlap(C.Structure):
  _fields_ = [('id', C.c_int32), ('other_id', C.c_int32), ('count', C.c_int64)]


class SeedPolicyDesc(C.Structure):
  _fields_ = [('kind', C.c_int32), ('min_distance', C.c_int32), ('threshold_abs', C.c_double),
              ('threshold_abs_is_min', C.c_int32), ('use_threshold_rel', C.c_int32), ('threshold_rel', C.c_double)]


class DecisionPointDesc(C.Structure):
  _fields_ = [('shape_zyx', C.c_int32 * 3), ('voxel_size_xyz', C.c_int32 * 3), ('use_max_distance', C.c_int32),
              ('reserved', C.c_int32), ('max_distance', C.c_double), ('box_start_zyx', C.c_int32 * 3),
              ('box_size_zyx', C.c_int32 * 3), ('dust_threshold', C.c_int64)]


class ExclusionSphere(C.Structure):
  _fields_ = [('c_xyz', C.c_int64 * 3), ('r2', C.c_int64), ('f_xyz', C.c_double * 3), ('f_r2', C.c_double),
              ('integer', C.c_int32), ('reserved', C.c_int32)]


class PartitionDesc(C.Structure):
  _fields_ = [('shape_zyx', C.c_int32 * 3), ('lom_radius_zyx', C.c_int32 * 3), ('min_size', C.c_int64),
              ('thresholds', C.c_void_p), ('n_thresholds', C.c_int32), ('use_whitelist', C.c_int32),
              ('whitelist', C.c_void_p), ('n_whitelist', C.c_int64), ('spheres', C.c_void_p),
              ('n_spheres', C.c_int32), ('reserved', C.c_int32), ('scratch_bytes', C.c_int64),
              ('n_labels_out', C.c_void_p)]


class PartitionRowsDesc(C.Structure):
  _fields_ = [('shape_zyx', C.c_int32 * 3), ('crop_start_zyx', C.c_int32 * 3), ('crop_shape_zyx', C.c_int32 * 3),
              ('reserved', C.c_int32), ('volume_index', C.c_int64)]


class TrainDesc(C.Structure):
  _fields_ = [('optimizer', C.c_int32), ('momentum', C.c_float), ('beta1', C.c_float), ('beta2', C.c_float),
              ('epsilon', C.c_float), ('max_gradient_entry_mag', C.c_float), ('max_batch', C.c_int32)]


FOV_POLICIES = {'fixed': 0, 'max_pred_moves': 1}   # FFN_FOV_*
# FfnExampleCoord, as a numpy record so that a stream of them is one contiguous array
EXAMPLE_COORD_DTYPE = np.dtype([('volume', '<i4'), ('center_xyz', '<i4', (3,)), ('permutation_zyx', '<i4', (3,)),
                                ('reflect_zyx', '<i4', (3,))])


class ExampleVolume(C.Structure):
  _fields_ = [('image', C.c_void_p), ('labels', C.c_void_p), ('image_shape_zyx', C.c_int32 * 3),
              ('label_shape_zyx', C.c_int32 * 3), ('offset', C.c_float), ('scale', C.c_float)]


class ExampleDesc(C.Structure):
  _fields_ = [('policy', C.c_int32), ('fov_moves', C.c_int32), ('seed_pad', C.c_float), ('seed_logit_pad', C.c_float),
              ('seed_logit_centre', C.c_float), ('batch', C.c_int32), ('seed_threshold', C.c_double),
              ('label_threshold', C.c_double), ('shifts_zyx', C.c_void_p), ('n_shifts', C.c_int32),
              ('permutable_zyx', C.c_int32 * 3), ('reflectable_zyx', C.c_int32 * 3), ('eval_threshold', C.c_double)]


class TrackerCounts(C.Structure):
  _fields_ = [('steps', C.c_int64), ('patches', C.c_int64), ('eval_voxels', C.c_int64),
              ('prediction_counts', C.c_int64 * 4), ('patch_loss', C.c_double)]


class CleanUpDesc(C.Structure):
  _fields_ = [('shape_zyx', C.c_int32 * 3), ('connectivity', C.c_int32), ('min_size', C.c_int64)]


class CoordinateVolume(C.Structure):
  _fields_ = [('crop_shape_zyx', C.c_int32 * 3), ('margin_zyx', C.c_int32 * 3), ('name_offset', C.c_int64),
              ('name_length', C.c_int64)]


class CoordinateDesc(C.Structure):
  _fields_ = [('volumes', C.c_void_p), ('n_volumes', C.c_int32), ('reserved', C.c_int32), ('names', C.c_void_p),
              ('names_bytes', C.c_int64)]


# FfnDecisionPoint, as a numpy record so that the output array is filled in place
DECISION_POINT_DTYPE = np.dtype([('id_a', '<u8'), ('id_b', '<u8'), ('dist', '<f8'), ('point_xyz', '<i8', (3,))])


class ResegEvalDesc(C.Structure):
  _fields_ = [('box_zyx', C.c_int32 * 3), ('voxel_size_zyx', C.c_int32 * 3), ('pair', C.c_int32),
              ('reserved', C.c_int32), ('num_items', C.c_int64)]


# FfnResegStats and FfnResegOverlap, as numpy records so that the output arrays are filled in place
RESEG_STATS_DTYPE = np.dtype([('n_seg', '<i8', (2,)), ('n_reseg', '<i8', (2,)), ('n_reseg_seg', '<i8', (2, 2)),
                              ('n_inter', '<i8'), ('n_union', '<i8'), ('max_edt2', '<u8', (4,))])
RESEG_OVERLAP_DTYPE = np.dtype([('item', '<i8'), ('id', '<u8'), ('num_overlapping', '<i8'), ('num_original', '<i8')])


class Counters(C.Structure):
  _fields_ = [(n, C.c_int64) for n in (
      'inference_calls', 'segment_at_calls', 'seeds_examined', 'skip_threshold', 'skip_invalid_pos',
      'skip_restricted_pos', 'seed_got_too_weak', 'voxels_segmented', 'voxels_overlapping',
      'invalid_weak', 'invalid_small', 'invalid_other', 'segments', 'max_id')] + [
          ('device_seconds', C.c_double), ('kernel_launches', C.c_int64)]


_lib = None


def build_if_needed():
  from . import build as _build
  return _build.build()


def load() -> C.CDLL:
  """Loads (building first when nvcc is available and sources are newer) the engine library."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    try:
      build_if_needed()
    except Exception as e:  # pylint: disable=broad-except
      raise ImportError(
          'libffn_b200.so is missing and could not be built (%s). The FFN engine has no CPU '
          'fallback.' % e) from e
  lib = C.CDLL(LIB_PATH)
  p = C.c_void_p
  i32p = C.POINTER(C.c_int32)
  lib.ffn_last_error.restype = C.c_char_p
  lib.ffn_last_error.argtypes = []
  lib.ffn_engine_create.argtypes = [C.c_int, C.POINTER(ModelDesc), C.POINTER(C.c_void_p),
                                    C.POINTER(C.c_void_p), C.c_int, C.POINTER(p)]
  lib.ffn_engine_destroy.argtypes = [p]
  lib.ffn_engine_destroy.restype = None
  lib.ffn_engine_set_compute_mode.argtypes = [p, C.c_int]
  lib.ffn_engine_set_grid.argtypes = [p, C.c_int]
  lib.ffn_engine_set_chains.argtypes = [p, C.c_int]
  lib.ffn_engine_set_step_chunk.argtypes = [p, C.c_int64]
  lib.ffn_engine_info.argtypes = [p, C.POINTER(C.c_int64)]
  lib.ffn_engine_profile.argtypes = [p, C.POINTER(C.c_int64), C.c_int]
  lib.ffn_engine_trace.argtypes = [p, C.POINTER(C.c_int64), C.c_int64, C.c_int]
  lib.ffn_face_table.argtypes = [C.POINTER(ModelDesc), C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_int64),
                                 C.POINTER(C.c_int32), C.POINTER(C.c_int64)]
  lib.ffn_predict.argtypes = [p, p, p, C.c_int, p]
  lib.ffn_canvas_create.argtypes = [p, p, C.c_int, i32p, C.c_float, C.c_float, C.POINTER(Options),
                                    C.c_int, C.POINTER(p)]
  lib.ffn_canvas_destroy.argtypes = [p]
  lib.ffn_canvas_destroy.restype = None
  lib.ffn_canvas_set_mask.argtypes = [p, C.c_int, p]
  lib.ffn_canvas_segment_at.argtypes = [p, i32p, C.c_int, C.c_int64, C.POINTER(SegStats)]
  lib.ffn_canvas_segment_all.argtypes = [p, p, C.c_int64, p, C.c_int64, C.POINTER(C.c_int64), p,
                                         C.c_int64, C.POINTER(C.c_int64), C.POINTER(Counters)]
  lib.ffn_canvas_update_at.argtypes = [p, i32p, p]
  lib.ffn_canvas_init_seed.argtypes = [p, i32p]
  lib.ffn_canvas_read.argtypes = [p, C.c_int, i32p, i32p, p]
  lib.ffn_canvas_write.argtypes = [p, C.c_int, i32p, i32p, p]
  lib.ffn_canvas_policy_state_size.argtypes = [p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
  lib.ffn_canvas_policy_state_get.argtypes = [p, p, p, i32p]
  lib.ffn_canvas_policy_state_set.argtypes = [p, p, C.c_int64, p, C.c_int64, i32p]
  lib.ffn_canvas_set_resume.argtypes = [p, C.c_int64, i32p, i32p]
  lib.ffn_canvas_trace.argtypes = [p, C.c_int64, p, C.POINTER(C.c_int64)]
  lib.ffn_canvas_seed_peaks.argtypes = [p, C.POINTER(C.c_float), p, p, C.c_int64, C.POINTER(C.c_int64)]
  lib.ffn_canvas_seed_policy.argtypes = [p, C.POINTER(SeedPolicyDesc), p, p, C.c_int64, C.POINTER(C.c_int64)]
  lib.ffn_canvas_set_max_id.argtypes = [p, C.c_int64]
  lib.ffn_canvas_get_counters.argtypes = [p, C.POINTER(Counters)]
  lib.ffn_canvas_spec_stats.argtypes = [p, C.POINTER(C.c_int64)]
  lib.ffn_canvas_sched_stats.argtypes = [p, C.POINTER(C.c_int64), C.c_int]
  lib.ffn_canvas_device_ptr.argtypes = [p, C.c_int, C.POINTER(p), C.POINTER(C.c_int64)]
  lib.ffn_canvas_add_id_offset.argtypes = [p, C.c_int32]
  lib.ffn_decision_points.argtypes = [C.c_int, C.POINTER(DecisionPointDesc), p, p, C.c_int64, C.POINTER(C.c_int64)]
  lib.ffn_reseg_eval.argtypes = [C.c_int, C.POINTER(ResegEvalDesc), p, p, p, p, p, p, C.c_int64, C.POINTER(C.c_int64)]
  lib.ffn_split_intersection.argtypes = [C.c_int, C.c_int64, p, p, C.c_int64]
  lib.ffn_compute_partitions.argtypes = [C.c_int, C.POINTER(PartitionDesc), p, p, p, p]
  lib.ffn_partition_rows.argtypes = [C.c_int, C.POINTER(PartitionRowsDesc), p, p, p]
  lib.ffn_coordinate_records.argtypes = [C.c_int, C.POINTER(CoordinateDesc), p, C.c_int64, p, C.c_int64,
                                         C.POINTER(C.c_int64)]
  lib.ffn_clean_up.argtypes = [C.c_int, C.POINTER(CleanUpDesc), p, p, p, p, C.c_int64, C.POINTER(C.c_int64)]
  lib.ffn_trainer_create.argtypes = [C.c_int, C.POINTER(ModelDesc), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                     C.POINTER(TrainDesc), C.POINTER(p)]
  lib.ffn_trainer_destroy.argtypes = [p]
  lib.ffn_trainer_destroy.restype = None
  lib.ffn_trainer_step.argtypes = [p, p, p, p, p, C.c_int, C.c_float, p, C.POINTER(C.c_double)]
  lib.ffn_trainer_gradients.argtypes = [p, p, p, p, p, C.c_int, p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                        C.POINTER(C.c_double)]
  lib.ffn_trainer_get_weights.argtypes = [p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]
  lib.ffn_trainer_train.argtypes = [p, p, p, C.c_int64, C.c_int, p, p, C.POINTER(C.c_int64)]
  lib.ffn_examples_create.argtypes = [C.c_int, C.POINTER(ModelDesc), C.POINTER(ExampleDesc), p, C.c_int, C.POINTER(p)]
  lib.ffn_examples_destroy.argtypes = [p]
  lib.ffn_examples_destroy.restype = None
  lib.ffn_examples_next.argtypes = [p, p, C.c_int64, p, p, p, p, p, C.POINTER(C.c_int64)]
  lib.ffn_examples_update.argtypes = [p, p]
  lib.ffn_examples_read_seeds.argtypes = [p, p]
  lib.ffn_examples_tracker.argtypes = [p, C.POINTER(TrackerCounts), p, C.c_int, p, p, C.POINTER(C.c_int32), C.c_int]
  lib.ffn_selftest_wgmma.argtypes = [C.c_int, C.POINTER(C.c_double), C.c_int]
  for name in EXPORTS:
    if name not in ('ffn_last_error', 'ffn_engine_destroy', 'ffn_canvas_destroy', 'ffn_trainer_destroy',
                    'ffn_examples_destroy'):
      getattr(lib, name).restype = C.c_int
  _lib = lib
  return lib


def check(rc: int):
  if rc != 0:
    raise RuntimeError(load().ffn_last_error().decode('utf-8', 'replace'))


def i3(v):
  return (C.c_int32 * 3)(int(v[0]), int(v[1]), int(v[2]))


def ptr(a: np.ndarray):
  return a.ctypes.data_as(C.c_void_p)
