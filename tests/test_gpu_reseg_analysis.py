"""Resegmentation analysis on the device (ffn_reseg_eval): protos equal, field by field, to the ones the reference's
own module wrote (tests/golden/reseg_analysis_ref.npz), batches equal to single calls, the oracle at size on a
configs[4]-like volume, and a result file written by this package's process_point."""
import os

import numpy as np
import pytest

from ffn_b200.inference import resegmentation_analysis as ra
from oracle import reseg_analysis as ora
from test_reseg_analysis import fixture_cases

pytestmark = pytest.mark.gpu


def _single(case):
  tag, kind, path, vol, radius, analysis, voxel, threshold, _, _ = case
  if kind == 'pair':
    return ra.evaluate_pair_resegmentation(path, vol, radius, analysis, voxel, threshold)
  return ra.evaluate_endpoint_resegmentation(path, vol, radius, threshold)


def test_device_equals_reference_fixture(tmp_path):
  for case in fixture_cases(tmp_path):
    tag, kind, path, vol, radius, analysis, voxel, threshold, expect, error = case
    if error:
      with pytest.raises(getattr(ra, error)):
        _single(case)
      continue
    got = _single(case)
    want = type(got).FromString(expect)
    assert got == want, (tag, got, want)          # every field, floats with ==
    assert got.SerializeToString(deterministic=True) == expect, tag
    # the volume store form of the segmentation reads the same boxes
    store = type('Store', (), {'__getitem__': lambda self, ind: vol[(slice(ind[0], ind[0] + 1),) + tuple(ind[1:])]})()
    if kind == 'pair':
      again = ra.evaluate_pair_resegmentation(path, store, radius, analysis, voxel, threshold)
    else:
      again = ra.evaluate_endpoint_resegmentation(path, store, radius, threshold)
    assert again == got, tag


def test_batch_equals_single_items(tmp_path):
  cases = fixture_cases(tmp_path)
  groups = {}
  for c in cases:
    groups.setdefault((c[1], c[3].shape, c[4], c[5], c[6], c[7]), []).append(c)
  assert any(len(g) > 2 for g in groups.values())
  for (kind, _, radius, analysis, voxel, threshold), group in groups.items():
    paths = [c[2] for c in group] * 2
    vol = group[0][3]
    if kind == 'pair':
      batch = ra.evaluate_pair_resegmentations(paths, vol, radius, analysis, voxel, threshold)
    else:
      batch = ra.evaluate_endpoint_resegmentations(paths, vol, radius, threshold)
    assert len(batch) == len(paths)
    for c, got in zip(group * 2, batch):
      if c[9]:
        assert isinstance(got, getattr(ra, c[9])), c[0]
      else:
        assert got == _single(c) and got.SerializeToString(deterministic=True) == c[8], c[0]


def test_evaluate_segmentation_result_on_device():
  from ffn_b200.inference import resegmentation_pb2
  from scipy import ndimage
  rng = np.random.RandomState(3)
  seg = rng.randint(0, 3, (9, 15, 17))
  reseg = ndimage.binary_dilation(seg == 1)
  moves = rng.randint(0, 12, (20, 3))
  dels = rng.randint(0, 50, 20)
  got = resegmentation_pb2.PairResegmentationResult.SegmentResult()
  ra.evaluate_segmentation_result(reseg, dels, moves, (1, 2, 3), (4, 6, 7), seg == 1, seg == 2, (3, 2, 5), got)
  want = resegmentation_pb2.PairResegmentationResult.SegmentResult()
  ora._segment_result(reseg, dels, moves, (1, 2, 3), (4, 6, 7), seg == 1, seg == 2, (3, 2, 5), want)
  assert got == want
  # an object that fills the box: no background voxel for the distance transform, scipy's value all the same
  full = np.ones(seg.shape, bool)
  got = resegmentation_pb2.PairResegmentationResult.SegmentResult()
  ra.evaluate_segmentation_result(full, dels, moves, (1, 2, 3), (4, 6, 7), seg == 1, seg == 2, (3, 2, 5), got,
                                  device=0)
  want = resegmentation_pb2.PairResegmentationResult.SegmentResult()
  ora._segment_result(full, dels, moves, (1, 2, 3), (4, 6, 7), seg == 1, seg == 2, (3, 2, 5), want)
  assert got == want and got.num_voxels == full.size


def test_batch_at_size_equals_oracle(tmp_path):
  """A few hundred decision points of a configs[4]-like Voronoi volume (voxel size (40, 16, 16)) at the manual's
  analysis radius, with synthetic result files: one device batch against the scipy oracle."""
  from ffn_b200 import synthetic
  from ffn_b200.utils import decision_point as dp
  _, cells = synthetic.voronoi_phantom((128, 256, 256), seed=3, voxel_size_zyx=(2.5, 1.0, 1.0), cell_volume=20000.0,
                                       return_cells=True)
  seg = cells.astype(np.uint64)
  seg[seg > 0] += np.uint64(2**63 - 1000)
  points = dp.find_decision_points(seg, (16, 16, 40))
  radius, analysis, voxel = (20, 40, 40), (17, 34, 34), (40, 16, 16)
  rng = np.random.RandomState(0)
  keys = list(points)
  picked = [keys[i] for i in rng.permutation(len(keys))]
  items = [(a, b, tuple(int(v) for v in points[(a, b)][1])) for a, b in picked]
  fits = lambda xyz: all(r <= c < n - r for c, r, n in zip(xyz[::-1], radius, seg.shape))  # noqa: E731
  items = [it for it in items if fits(it[2])][:240]
  paths = ora.write_synthetic_results(seg, items, radius, str(tmp_path), seed=1)
  assert len(paths) == 240, len(paths)
  vol = seg[np.newaxis]
  got = ra.evaluate_pair_resegmentations(paths, vol, radius, analysis, voxel)
  for path, g in zip(paths, got):
    try:
      want = ora.evaluate_pair_resegmentation(path, vol, radius, analysis, voxel)
    except ora.InvalidBaseSegmentatonError:
      assert isinstance(g, ra.InvalidBaseSegmentatonError), path
      continue
    assert g == want, (path, g, want)
  assert sum(not isinstance(g, Exception) for g in got) >= 150
  ends = paths[:40]   # scored as endpoints of their first object
  got_e = ra.evaluate_endpoint_resegmentations(ends, vol, radius)
  for path, g in zip(ends, got_e):
    assert g == ora.evaluate_endpoint_resegmentation(path, vol, radius), path


def test_result_file_written_by_process_point(tmp_path, golden_dir):
  """A pair point resegmented by this package's process_point (Runner + device canvas), scored through both
  ffn_b200.inference and ffn.inference, equals the oracle."""
  from google.protobuf import text_format
  from ffn.inference import inference_pb2, resegmentation, runner as runner_mod
  from ffn.inference import resegmentation_analysis as ffn_ra
  from ffn_b200 import synthetic
  vol, cells = synthetic.voronoi_phantom((64, 64, 64), seed=7, cell_volume=30000.0, return_cells=True)
  np.save(tmp_path / 'vol.npy', vol)
  seg = cells[np.newaxis].astype(np.uint64)
  np.save(tmp_path / 'seg.npy', seg)
  found = None
  for z in range(28, 37):
    for y in range(28, 37):
      for x in range(28, 37):
        if found is None and cells[z, y, x] == 0:
          left = [int(v) for v in cells[z, y, x - 4:x][::-1] if v > 0]
          right = [int(v) for v in cells[z, y, x + 1:x + 5] if v > 0]
          if left and right and left[0] != right[0]:
            found = (z, y, x, left[0], right[0])
  assert found is not None
  z, y, x, id_a, id_b = found
  req = inference_pb2.ResegmentationRequest()
  text_format.Parse('''inference { image { hdf5: "%s:raw" } init_segmentation { hdf5: "%s:seg" }
      image_mean: 128 image_stddev: 33 model_checkpoint_path: "%s" model_name: "convstack_3d.ConvStack3DFFNModel"
      model_args: "{\\"depth\\": 12, \\"fov_size\\": [33, 33, 33], \\"deltas\\": [8, 8, 8]}"
      segmentation_output_dir: "%s"
      inference_options { init_activation: 0.95 pad_value: 0.05 move_threshold: 0.9 min_boundary_dist { x: 1 y: 1 z: 1}
                          segment_threshold: 0.6 min_segment_size: 1000 } }
      radius { x: 24 y: 24 z: 24 } output_directory: "%s" max_retry_iters: 2
      exclusion_radius { x: 4 y: 4 z: 4 } analysis_radius { x: 16 y: 16 z: 16 }''' % (
          tmp_path / 'vol.npy', tmp_path / 'seg.npy', os.path.join(golden_dir, 'fib25_convstack.npz'),
          tmp_path / 'segout', tmp_path / 'reseg'), req)
  pt = req.points.add()
  pt.id_a, pt.id_b = id_a, id_b
  pt.point.x, pt.point.y, pt.point.z = x, y, z
  runner = runner_mod.Runner()
  runner.start(req.inference)
  resegmentation.process(req, runner)
  runner.stop_executor()
  path = str(tmp_path / 'reseg' / ('%d-%d_at_%d_%d_%d.npz' % (id_a, id_b, x, y, z)))
  args = (path, seg, (24, 24, 24), (16, 16, 16), (4, 3, 3))
  want = ora.evaluate_pair_resegmentation(*args, threshold=0.6)
  for module in (ra, ffn_ra):
    got = module.evaluate_pair_resegmentation(*args, threshold=0.6)
    assert got == want and got.eval.from_a.num_voxels > 0 and got.eval.from_b.num_voxels > 0
