"""PolicyPeaks2d / PolicyFillEmptySpace / PolicyMaxPeaks on the device (ffn_canvas_seed_policy): against the
reference's own policies (tests/golden/peak_policies_ref.npz), against the scipy host path on a larger anisotropic
phantom, and through Runner on the anisotropic geometry and on top of an init_segmentation."""

import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CASES = ['p2d_default', 'p2d_md3_desc', 'p2d_masked', 'fill', 'max_excl', 'max_rel']
KINDS = {'PolicyPeaks2d': 'peaks_2d', 'PolicyFillEmptySpace': 'fill_empty', 'PolicyMaxPeaks': 'max_peaks'}
MODEL_ARGS_ANISO = '{\\"depth\\": 12, \\"fov_size\\": [33, 33, 17], \\"deltas\\": [8, 8, 4]}'


def _image(vol):
  return (vol.astype(np.float32) - np.float32(128.0)) / np.float32(33.0)


@pytest.fixture(scope='module')
def ref(golden_dir):
  return np.load(os.path.join(golden_dir, 'peak_policies_ref.npz'))


@pytest.fixture(scope='module')
def engine(golden_dir):
  from ffn_b200 import engine as eng, tf_checkpoint
  w, b = tf_checkpoint.load_convstack_npz(os.path.join(golden_dir, 'fib25_convstack.npz'))
  e = eng.Engine(w, b, (33, 33, 33), (8, 8, 8))
  yield e
  e.close()


class _Restrictor:
  def __init__(self, mask=None, seed_mask=None):
    self.mask, self.seed_mask, self.shift_mask = mask, seed_mask, None


class _HostCanvas:
  """Just enough canvas for the host (scipy) path of the seed policies: no `_dev`."""

  def __init__(self, image, segmentation, restrictor, margin):
    self.image, self.segmentation, self.restrictor = image, segmentation, restrictor
    self.margin, self.shape, self.voxel_size_zyx = np.asarray(margin), image.shape, (1, 1, 1)


@pytest.mark.parametrize('case', CASES)
def test_device_peaks_equal_reference(engine, ref, case):
  """The device's raw peak list, border-filtered with the fixture's margin and sorted as the policy sorts, is the
  reference policy's list (u8 image normalised on the device, masks and segmentation resident)."""
  from ffn_b200 import _lib, engine as eng
  policy, kwargs = str(ref[case + '_policy']), json.loads(str(ref[case + '_kwargs']))
  vol = ref[case + '_volume']
  cv = eng.DeviceCanvas(engine, vol, eng.make_options(), 128.0, 33.0, keep_probability_maps=False)
  try:
    if case + '_mask' in ref:
      cv.set_mask(_lib.MASK_MOVEMENT, ref[case + '_mask'])
    if case + '_seed_mask' in ref:
      cv.set_mask(_lib.MASK_SEED, ref[case + '_seed_mask'])
    cv.write(_lib.ARRAY_SEGMENTATION, ref[case + '_segmentation'])
    rng = np.random.RandomState(seed=42)
    if policy == 'PolicyPeaks2d':
      md, thr, rel, noise = kwargs.get('min_distance', 7), kwargs.get('threshold_abs', 2.5), 0, rng.rand(*vol.shape[1:])
    elif policy == 'PolicyFillEmptySpace':
      md, thr, rel, noise = 2, 0.5, 0, rng.rand(*vol.shape)
    else:
      md, thr, rel = kwargs.get('min_distance', 3), kwargs.get('threshold_abs', 0), kwargs.get('threshold_rel', 0)
      noise = rng.rand(*vol.shape)
    raw = cv.seed_policy(KINDS[policy], md, thr, rel, noise).astype(np.int64)
    # a tiny output capacity is grown to the number of peaks
    np.testing.assert_array_equal(cv.seed_policy(KINDS[policy], md, thr, rel, noise, cap=1), raw)
  finally:
    cv.close()
  assert [tuple(r) for r in raw] == sorted(tuple(r) for r in raw)
  if kwargs.get('sort_cmp', 'ascending').startswith('de'):
    raw = raw[::-1]
  m = ref[case + '_margin'][None]
  got = raw[np.all((raw - m >= 0) & (raw + m < np.asarray(vol.shape)[None]), axis=1)]
  print('%s: device %d raw peaks, %d after the border filter, reference %d' % (
      case, raw.shape[0], got.shape[0], ref[case + '_coords'].shape[0]))
  np.testing.assert_array_equal(got, ref[case + '_coords'])


def test_device_equals_host_on_anisotropic_phantom(golden_dir):
  """48x160x176 serial-section phantom with a movement mask, a seed mask, labelled cells and -1 markers: the device
  path of every policy (through inference.Canvas) yields the host path's list."""
  from ffn.inference import executor, inference, inference_pb2, inference_utils, movement, seed as seed_mod
  from ffn.training.models import convstack_3d
  from ffn_b200 import synthetic
  shape = (48, 160, 176)
  vol, cells = synthetic.voronoi_phantom(shape, seed=21, sigma=(0.5, 1.0, 1.0), voxel_size_zyx=(4.0, 1.0, 1.0),
                                         cell_volume=20000.0, return_cells=True)
  rng = np.random.RandomState(22)
  mask = np.zeros(shape, dtype=bool)
  mask[:, :, :20] = True
  seed_mask = rng.rand(*shape) > 0.995
  seg = np.zeros(shape, dtype=np.int32)
  ids = np.unique(cells[cells > 0])
  for k, cid in enumerate(ids[rng.rand(ids.size) < 0.5]):
    seg[cells == cid] = k + 1
  seg[rng.randint(0, shape[0], 200), rng.randint(0, shape[1], 200), rng.randint(0, shape[2], 200)] = -1
  model = convstack_3d.ConvStack3DFFNModel(fov_size=[33, 33, 33], deltas=[8, 8, 8], depth=12)
  exe = executor.B200Executor(executor.ExecutorInterface(), model, inference_utils.Counters(),
                              checkpoint_path=os.path.join(golden_dir, 'fib25_convstack.npz'))
  opts = inference_pb2.InferenceOptions(init_activation=0.95, pad_value=0.05, move_threshold=0.9,
                                        segment_threshold=0.6, min_segment_size=1000)
  cv = inference.Canvas(model.info, exe.get_client(inference_utils.Counters()), vol, opts,
                        restrictor=movement.MovementRestrictor(mask=mask, seed_mask=seed_mask), voxel_size_zyx=(4, 1, 1),
                        image_mean=128, image_stddev=33)
  cv.segmentation[...] = seg
  host = _HostCanvas(_image(vol), seg, _Restrictor(mask, seed_mask), cv.margin)
  for name, kwargs in (('PolicyPeaks2d', {}), ('PolicyPeaks2d', {'min_distance': 3, 'threshold_abs': 0}),
                       ('PolicyFillEmptySpace', {}), ('PolicyMaxPeaks', {}),
                       ('PolicyMaxPeaks', {'threshold_abs': None, 'threshold_rel': 0.4, 'min_distance': 5})):
    got = getattr(seed_mod, name)(cv, **kwargs).remaining()
    want = getattr(seed_mod, name)(host, **kwargs).remaining()
    print('%s %r: device %d seeds, host %d' % (name, kwargs, got.shape[0], want.shape[0]))
    assert want.shape[0] > 20
    np.testing.assert_array_equal(got, want)
  exe.close()


def _request(tmp_path, golden_dir, policy, model_args, init_seg=False):
  from google.protobuf import text_format
  from ffn.inference import inference_pb2
  req = inference_pb2.InferenceRequest()
  text_format.Parse('''
    image { hdf5: "%s:raw" } %s
    image_mean: 128 image_stddev: 33 seed_policy: "%s"
    model_checkpoint_path: "%s"
    model_name: "convstack_3d.ConvStack3DFFNModel"
    model_args: "%s"
    segmentation_output_dir: "%s"
    inference_options { init_activation: 0.95 pad_value: 0.05 move_threshold: 0.9
                        min_boundary_dist { x: 1 y: 1 z: 1} segment_threshold: 0.6 min_segment_size: 100 }
  ''' % (tmp_path / 'vol.npy', ('init_segmentation { hdf5: "%s:seg" }' % (tmp_path / 'seg.npy')) if init_seg else '',
         policy, os.path.join(golden_dir, 'fib25_convstack.npz'), model_args, tmp_path / 'out'), req)
  return req


def test_runner_peaks2d_on_the_anisotropic_geometry(tmp_path, golden_dir):
  """Runner with seed_policy "PolicyPeaks2d", fov_size [33, 33, 17] and deltas [8, 8, 4] (xyz) on a serial-section
  phantom: the canvas consumes exactly the oracle's seed list and produces a segmentation."""
  from ffn.inference import runner as runner_mod, storage
  from ffn_b200 import synthetic
  from oracle import seed_policies
  shape = (32, 112, 112)
  vol = synthetic.voronoi_phantom(shape, seed=23, sigma=(0.5, 1.0, 1.0), voxel_size_zyx=(4.0, 1.0, 1.0),
                                  cell_volume=12000.0)
  np.save(tmp_path / 'vol.npy', vol)
  runner = runner_mod.Runner()
  runner.start(_request(tmp_path, golden_dir, 'PolicyPeaks2d', MODEL_ARGS_ANISO))
  canvas = runner.run((0, 0, 0), shape)
  runner.stop_executor()
  assert canvas is not None and tuple(canvas.margin) == (8, 16, 16)
  want = seed_policies.policy_peaks_2d(_image(vol), margin_zyx=canvas.margin)
  assert want.shape[0] > 10
  coords, idx = canvas.seed_policy.get_state()
  np.testing.assert_array_equal(np.asarray(coords), want)
  assert idx == want.shape[0]
  seg, origins = storage.load_segmentation(str(tmp_path / 'out'), (0, 0, 0))
  print('PolicyPeaks2d: %d seeds, %d objects, %d voxels labelled' % (want.shape[0], len(origins), int((seg > 0).sum())))
  assert len(origins) > 0 and (seg > 0).sum() > 0
  assert {tuple(o.start_zyx) for o in origins.values()} <= set(map(tuple, want.tolist()))


def test_runner_fill_empty_space_only_adds_labels_in_unlabelled_voxels(tmp_path, golden_dir):
  """Runner with init_segmentation and seed_policy "PolicyFillEmptySpace": the seeds are the oracle's (computed from
  the initial segmentation), the initial labels stay as they are and new labels appear only where there were none."""
  from ffn.inference import runner as runner_mod, storage
  from ffn_b200 import synthetic
  from oracle import seed_policies
  shape = (64, 80, 88)
  vol, cells = synthetic.voronoi_phantom(shape, seed=24, cell_volume=15000.0, return_cells=True)
  rng = np.random.RandomState(25)
  init = np.zeros(shape, dtype=np.int32)
  ids = np.unique(cells[cells > 0])
  for k, cid in enumerate(ids[rng.rand(ids.size) < 0.6]):
    init[cells == cid] = k + 1                             # contiguous ids: the canvas keeps them as they are
  np.save(tmp_path / 'vol.npy', vol)
  np.save(tmp_path / 'seg.npy', init[np.newaxis].astype(np.uint64))
  runner = runner_mod.Runner()
  runner.start(_request(tmp_path, golden_dir, 'PolicyFillEmptySpace',
                        '{\\"depth\\": 12, \\"fov_size\\": [33, 33, 33], \\"deltas\\": [8, 8, 8]}', init_seg=True))
  canvas = runner.run((0, 0, 0), shape)
  runner.stop_executor()
  assert canvas is not None
  want = seed_policies.policy_fill_empty_space(init, margin_zyx=canvas.margin)
  assert want.shape[0] > 3 and (init[tuple(want.T)] == 0).all()
  coords, idx = canvas.seed_policy.get_state()
  np.testing.assert_array_equal(np.asarray(coords), want)
  assert idx == want.shape[0]
  seg, origins = storage.load_segmentation(str(tmp_path / 'out'), (0, 0, 0))
  seg = seg.astype(np.int64)
  new = (seg > 0) & (init == 0)
  print('PolicyFillEmptySpace: %d seeds, %d new objects, %d voxels newly labelled' % (
      want.shape[0], len(origins), int(new.sum())))
  np.testing.assert_array_equal(seg[init > 0], init[init > 0])
  assert new.sum() > 0 and len(origins) > 0
  assert (seg[new] > init.max()).all()
