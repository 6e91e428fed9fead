"""The device seed policies against the scipy oracle over the sweep of seed_sweep_cases.py: the RAW peak lists of
ffn_canvas_seed_peaks (PolicyPeaks) and ffn_canvas_seed_policy (PolicyPeaks2d, PolicyFillEmptySpace,
PolicyMaxPeaks), before any canvas-margin filter, so that no margin can hide a peak at the array border.  Also the
device PolicyPeaks against the reference's own list (tests/golden/policy_peaks_ref.npz), and one Runner run whose
canvas margin (2 in z) is below PolicyPeaks' border of 3."""

import os

import numpy as np
import pytest

import seed_sweep_cases as sc

pytestmark = pytest.mark.gpu

KINDS = {'peaks_2d', 'fill_empty', 'max_peaks'}


@pytest.fixture(scope='module')
def engine(golden_dir):
  from ffn_b200 import engine as eng, tf_checkpoint
  w, b = tf_checkpoint.load_convstack_npz(os.path.join(golden_dir, 'fib25_convstack.npz'))
  e = eng.Engine(w, b, (33, 33, 33), (8, 8, 8))
  yield e
  e.close()


def _device(engine, c):
  """The device's raw, lexicographically sorted peak list for case `c`."""
  from ffn_b200 import _lib, engine as eng
  cv = eng.DeviceCanvas(engine, c['image'], eng.make_options(), c['mean'], c['std'], keep_probability_maps=False)
  try:
    if c['mask'] is not None:
      cv.set_mask(_lib.MASK_MOVEMENT, c['mask'])
    if c['seed_mask'] is not None:
      cv.set_mask(_lib.MASK_SEED, c['seed_mask'])
    cv.write(_lib.ARRAY_SEGMENTATION, c['segmentation'])
    if c['kind'] == 'peaks':
      got = cv.seed_peaks(c['voxel'], sc.noise(c))
    elif c['kind'] == 'fill_empty':
      got = cv.seed_policy('fill_empty', 2, 0.5, 0, sc.noise(c))
    else:
      got = cv.seed_policy(c['kind'], c['min_distance'], c['threshold_abs'], c['threshold_rel'], sc.noise(c))
  finally:
    cv.close()
  return sc.lexsorted(got)


@pytest.mark.parametrize('name', sc.NAMES)
def test_device_raw_peaks_equal_oracle(engine, name):
  c = sc.build(name)
  want = sc.oracle(c)
  got = _device(engine, c)
  print('%s (%s, %s): device %d raw peaks, oracle %d' % (name, c['kind'], c['image'].shape, got.shape[0], want.shape[0]))
  if c['exact_zero']:
    assert want.shape[0] == 0
  else:
    assert want.shape[0] >= sc.min_peaks(name)
  np.testing.assert_array_equal(got, want)


def _peaks_ref_cases():
  path = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'policy_peaks_ref.npz')
  with np.load(path) as r:
    return sorted(k[:-len('_coords')] for k in r.files if k.endswith('_coords'))


@pytest.mark.parametrize('case', _peaks_ref_cases())
def test_device_policy_peaks_equals_reference(engine, golden_dir, case):
  """ffn_canvas_seed_peaks followed by the canvas margin's border filter is the reference PolicyPeaks' list,
  including the canvases whose margin is below the peak border of 3."""
  from ffn_b200 import _lib, engine as eng
  r = np.load(os.path.join(golden_dir, 'policy_peaks_ref.npz'))
  vol = r[case + '_volume']
  cv = eng.DeviceCanvas(engine, vol, eng.make_options(), 128.0, 33.0, keep_probability_maps=False)
  try:
    if case + '_mask' in r.files:
      cv.set_mask(_lib.MASK_MOVEMENT, r[case + '_mask'])
      cv.set_mask(_lib.MASK_SEED, r[case + '_seed_mask'])
    cv.write(_lib.ARRAY_SEGMENTATION, r[case + '_segmentation'])
    raw = cv.seed_peaks(tuple(float(v) for v in r[case + '_voxel']), np.random.RandomState(seed=42).rand(*vol.shape))
  finally:
    cv.close()
  m = r[case + '_margin'][None]
  got = raw[np.all((raw - m >= 0) & (raw + m < np.asarray(vol.shape)[None]), axis=1)]
  want = r[case + '_coords']
  assert want.shape[0] >= 5
  np.testing.assert_array_equal(got, want)


def test_runner_policy_peaks_with_a_margin_below_the_peak_border(tmp_path, golden_dir):
  """Runner with seed_policy "PolicyPeaks", fov_size [33, 33, 5] and deltas [8, 8, 0] (xyz): the canvas margin is
  2 in z, so only the peak border keeps seeds off the z = 2 and z = Z - 3 planes.  The canvas consumes exactly the
  oracle's seed list."""
  from google.protobuf import text_format
  from ffn.inference import inference_pb2, runner as runner_mod
  from ffn_b200 import synthetic
  from oracle import seed_peaks
  shape = (24, 80, 88)
  vol = synthetic.voronoi_phantom(shape, seed=27, cell_volume=4000.0)
  np.save(tmp_path / 'vol.npy', vol)
  req = inference_pb2.InferenceRequest()
  text_format.Parse('''
    image { hdf5: "%s:raw" }
    image_mean: 128 image_stddev: 33 seed_policy: "PolicyPeaks"
    model_checkpoint_path: "%s"
    model_name: "convstack_3d.ConvStack3DFFNModel"
    model_args: "{\\"depth\\": 12, \\"fov_size\\": [33, 33, 5], \\"deltas\\": [8, 8, 0]}"
    segmentation_output_dir: "%s"
    inference_options { init_activation: 0.95 pad_value: 0.05 move_threshold: 0.9
                        min_boundary_dist { x: 1 y: 1 z: 1} segment_threshold: 0.6 min_segment_size: 100 }
  ''' % (tmp_path / 'vol.npy', os.path.join(golden_dir, 'fib25_convstack.npz'), tmp_path / 'out'), req)
  runner = runner_mod.Runner()
  runner.start(req)
  canvas = runner.run((0, 0, 0), shape)
  runner.stop_executor()
  assert canvas is not None and tuple(canvas.margin) == (2, 16, 16)
  image = (vol.astype(np.float32) - np.float32(128.0)) / np.float32(33.0)
  want = seed_peaks.policy_peaks(image, margin_zyx=canvas.margin)
  assert want.shape[0] > 10
  coords, idx = canvas.seed_policy.get_state()
  print('PolicyPeaks with margin %r: %d seeds' % (tuple(canvas.margin), want.shape[0]))
  np.testing.assert_array_equal(np.asarray(coords), want)
  assert idx == want.shape[0]
