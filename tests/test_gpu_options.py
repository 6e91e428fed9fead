"""The device flood-fill loop away from the FIB-25 inference options, against the hybrid oracle.

The same option cases as tests/golden/make_golden_options.py (whose reference runs pin the CPU oracle,
tests/test_oracle_golden.py::test_toy_flood_fill_at_other_inference_options), here on the FIB-25 network: the
oracle loop driven by the GPU's own network ("hybrid oracle") and the persistent kernel must agree bit for bit
on seed, labels, origins, overlaps and counters (qprob within +-1 LSB, expf vs scipy expit at bin edges).
Every case also asserts, on the hybrid oracle, that it reaches the path it is there for: the disco merge
switched off, applied on some steps only or never, a movement-policy threshold below / above the move
threshold, a seed that gets too weak.  The InferenceRequest / Canvas tests check that the options reach the
device through the public Python API.
"""

import json
import os

import numpy as np
import pytest

from oracle import flood_fill as ff

pytestmark = pytest.mark.gpu

FOV, DELTAS = (33, 33, 33), (8, 8, 8)
MOVE = ff.policy_threshold(0.9)

# probability-space InferenceOptions over the FIB-25 defaults of ff.Options; 'policy_score_threshold' is the
# movement policy's score_threshold (logit space), 'disco_partial' is filled in from the default run
CASES = {
    'default': {},
    'manual': dict(pad_value=0.5, move_threshold=0.6, segment_threshold=0.6, min_boundary_dist=(1, 2, 2),
                   min_segment_size=1000),
    'disco_off': dict(disco_seed_threshold=-1.0),
    'disco_partial': None,
    'disco_never': dict(disco_seed_threshold=1.0),
    'policy_low': dict(policy_score_threshold=MOVE - 2.0),
    'policy_high': dict(policy_score_threshold=MOVE + 1.5),
    'seg_low_pad_low': dict(segment_threshold=0.2, pad_value=0.001),
    'seg_high_move_high': dict(segment_threshold=0.97, move_threshold=0.97, init_activation=0.99),
    'weak_seed': dict(init_activation=0.91),
    'small_and_tight': dict(min_boundary_dist=(0, 0, 0), min_segment_size=0),
}


@pytest.fixture(scope='module')
def weights(golden_dir):
  from ffn_b200 import tf_checkpoint
  return tf_checkpoint.load_convstack_npz(os.path.join(golden_dir, 'fib25_convstack.npz'))


@pytest.fixture(scope='module')
def engines(weights):
  from ffn_b200 import _lib, engine as eng
  w, b = weights
  out = {'tc': eng.Engine(w, b, FOV, DELTAS, compute_mode=_lib.COMPUTE_FP16_TC),
         'fp32': eng.Engine(w, b, FOV, DELTAS, compute_mode=_lib.COMPUTE_FP32)}
  yield out
  for e in out.values():
    e.close()


@pytest.fixture(scope='module')
def g64(golden_dir):
  return np.load(os.path.join(golden_dir, 'flood_fill_64.npz'))


def _image(vol):
  return (vol.astype(np.float32) - np.float32(128.0)) / np.float32(33.0)


def _volume(name, g64):
  """(volume, seeds): the golden 64x72x80 volume and its grid seeds; weak_seed needs seeds that start on
  membranes, which a denser grid on a phantom provides."""
  if name == 'weak_seed':
    from ffn_b200.synthetic import voronoi_phantom
    vol = voronoi_phantom((64, 72, 80), seed=7, cell_volume=20000.0)
    return vol, ff.grid_seeds(vol.shape, step=8, offsets=(0, 4))
  return g64['volume'], g64['seeds']


def _hybrid(e, vol, seeds, opts, keep_probability_maps=True):
  """The oracle loop with the device's network; records mean(logits >= move) of every step."""
  fractions = []
  move = ff.f32_logit(opts.move_threshold)

  def net(seed, image):
    logits = e.predict(seed, image)
    fractions.append(float(np.mean(logits >= move)))
    return logits
  hyb = ff.Canvas(net, _image(vol), FOV, DELTAS, opts, keep_probability_maps=keep_probability_maps)
  hyb.segment_all(seeds)
  hyb.fractions = fractions
  return hyb


@pytest.fixture(scope='module')
def default_run(engines, g64):
  return _hybrid(engines['tc'], g64['volume'], g64['seeds'], ff.Options())


def _partial_threshold(fractions):
  """A disco_seed_threshold between two neighbouring per-step fractions of a run, near their median."""
  f = np.unique(np.float32(fractions))
  assert f.size >= 10
  mid = f.size // 2
  return float(np.float32((float(f[mid - 1]) + float(f[mid])) / 2))


@pytest.fixture(scope='module')
def disco_partial(default_run):
  return _partial_threshold(default_run.fractions)


def _options(name, disco_partial):
  over = dict(disco_seed_threshold=disco_partial) if name == 'disco_partial' else dict(CASES[name])
  return ff.Options(**over)


def _device_options(opts):
  from ffn_b200 import engine as eng
  return eng.make_options(init_activation=opts.init_activation, pad_value=opts.pad_value,
                          move_threshold=opts.move_threshold, segment_threshold=opts.segment_threshold,
                          disco_seed_threshold=opts.disco_seed_threshold, min_boundary_dist_zyx=opts.min_boundary_dist,
                          min_segment_size=opts.min_segment_size, policy_score_threshold=opts.policy_score_threshold)


def _device(e, vol, seeds, opts, chains, keep_probability_maps=True):
  from ffn_b200 import _lib, engine as eng
  e.set_chains(chains)
  try:
    cv = eng.DeviceCanvas(e, vol, _device_options(opts), 128.0, 33.0, keep_probability_maps=keep_probability_maps)
    origins, overlaps, ctr = cv.segment_all(seeds)
    out = dict(seg=cv.read(_lib.ARRAY_SEGMENTATION), seed=cv.read(_lib.ARRAY_SEED),
               qprob=cv.read(_lib.ARRAY_QPROB) if keep_probability_maps else None,
               origins=[(o.id, tuple(o.start_zyx), o.iters) for o in origins],
               overlaps=sorted((o.id, o.other_id, o.count) for o in overlaps),
               ctr={n: getattr(ctr, n) for n, _ in ctr._fields_ if n not in ('device_seconds', 'kernel_launches')})
    cv.close()
  finally:
    e.set_chains(0)
  return out


def _check_vs_hybrid(dev, hyb):
  np.testing.assert_array_equal(dev['seg'], hyb.segmentation)
  np.testing.assert_array_equal(dev['seed'], hyb.seed)
  if hyb.seg_prob is not None:
    qd = np.abs(dev['qprob'].astype(int) - hyb.seg_prob.astype(int))
    assert qd.max() <= 1 and (qd > 0).mean() < 1e-3
  assert dev['origins'] == [(k, v[0], v[1]) for k, v in sorted(hyb.origins.items())]
  assert dev['overlaps'] == sorted((k, int(i), int(c)) for k, v in hyb.overlaps.items() for i, c in zip(*v.tolist()))
  ctr = dev['ctr']
  for mine, theirs in (('inference_calls', 'inference-calls'), ('skip_threshold', 'skip_threshold'),
                       ('skip_invalid_pos', 'skip_invalid_pos'), ('seed_got_too_weak', 'seed_got_too_weak'),
                       ('invalid_weak', 'invalid-weak'), ('invalid_small', 'invalid-small'),
                       ('voxels_segmented', 'voxels-segmented'), ('voxels_overlapping', 'voxels-overlapping')):
    assert ctr[mine] == hyb.counters[theirs], mine
  assert ctr['inference_calls'] == len(hyb.trace)


def _check_reached(name, hyb, default_run):
  applied = np.asarray(hyb.disco_applied, dtype=bool)
  steps = len(hyb.trace)
  if name == 'manual':
    assert len(hyb.origins) >= 3
  elif name in ('disco_off', 'disco_never'):
    assert not applied.any() and steps > 0
  elif name == 'disco_partial':
    assert applied.sum() >= 5 and (~applied).sum() >= 5, (applied.sum(), (~applied).sum())
  elif name == 'policy_low':
    assert hyb.counters['skip_threshold'] > default_run.counters['skip_threshold']
  elif name == 'policy_high':
    assert 0 < steps < len(default_run.trace)
  elif name == 'weak_seed':
    assert hyb.counters['seed_got_too_weak'] > 0 and hyb.counters['invalid-weak'] > 0
  else:
    assert steps > 0


@pytest.mark.parametrize('name', list(CASES))
def test_device_loop_vs_hybrid_oracle_at_inference_options(engines, g64, default_run, disco_partial, name):
  """fp16 tensor-core mode: one chain bit-exact against the hybrid oracle; two and four chains bit-identical
  to one chain."""
  e = engines['tc']
  vol, seeds = _volume(name, g64)
  opts = _options(name, disco_partial)
  hyb = default_run if name == 'default' else _hybrid(e, vol, seeds, opts)
  _check_reached(name, hyb, default_run)
  one = _device(e, vol, seeds, opts, 1)
  _check_vs_hybrid(one, hyb)
  for chains in (2, 4):
    many = _device(e, vol, seeds, opts, chains)
    for k in ('seg', 'seed', 'qprob'):
      np.testing.assert_array_equal(many[k], one[k], err_msg='%d chains: %s' % (chains, k))
    for k in ('origins', 'overlaps', 'ctr'):
      assert many[k] == one[k], (chains, k)


@pytest.mark.parametrize('name', ['disco_partial', 'manual', 'seg_low_pad_low'])
def test_fp32_device_loop_vs_hybrid_oracle_at_inference_options(engines, g64, disco_partial, name):
  """The fp32 CUDA-core mode has its own epilogue and step count: same comparison, its own network."""
  e = engines['fp32']
  vol, seeds = _volume(name, g64)
  opts = _options(name, disco_partial)
  hyb = _hybrid(e, vol, seeds, opts)
  if name == 'disco_partial':
    applied = np.asarray(hyb.disco_applied, dtype=bool)
    assert applied.any() and not applied.all()
  _check_vs_hybrid(_device(e, vol, seeds, opts, 0), hyb)


def test_without_probability_maps(engines, g64, disco_partial):
  """keep_probability_maps=False changes nothing but the missing map."""
  e = engines['tc']
  vol, seeds = _volume('small_and_tight', g64)
  opts = _options('small_and_tight', disco_partial)
  kept = _device(e, vol, seeds, opts, 0)
  bare = _device(e, vol, seeds, opts, 0, keep_probability_maps=False)
  assert bare['qprob'] is None
  np.testing.assert_array_equal(bare['seg'], kept['seg'])
  np.testing.assert_array_equal(bare['seed'], kept['seed'])
  assert bare['origins'] == kept['origins'] and bare['ctr'] == kept['ctr']
  hyb = _hybrid(e, vol, seeds, opts, keep_probability_maps=False)
  _check_vs_hybrid(bare, hyb)


def test_runner_passes_every_option_to_the_device(tmp_path, golden_dir, g64, engines):
  """InferenceRequest -> Runner -> seg-*.npz with the manual's options, a partial disco threshold and a
  movement-policy threshold of its own: equal to the hybrid oracle run with the same options."""
  import dataclasses
  from google.protobuf import text_format
  from ffn.inference import inference_pb2, runner as runner_mod, storage
  from ffn_b200 import _lib
  score = 1.5                                     # logit(0.6) = 0.405
  seeds = ff.grid_seeds(g64['volume'].shape)      # PolicyGrid3d
  opts = ff.Options(pad_value=0.5, move_threshold=0.6, segment_threshold=0.6, min_boundary_dist=(1, 2, 2),
                    min_segment_size=1500, policy_score_threshold=score)
  disco_partial = _partial_threshold(_hybrid(engines['tc'], g64['volume'], seeds, opts).fractions)
  opts = dataclasses.replace(opts, disco_seed_threshold=disco_partial)
  vol_path = str(tmp_path / 'vol.npy')
  np.save(vol_path, g64['volume'])
  req = inference_pb2.InferenceRequest()
  text_format.Parse('''
    image { hdf5: "%s:raw" }
    image_mean: 128 image_stddev: 33 seed_policy: "PolicyGrid3d"
    model_checkpoint_path: "%s"
    model_name: "convstack_3d.ConvStack3DFFNModel"
    model_args: "{\\"depth\\": 12, \\"fov_size\\": [33, 33, 33], \\"deltas\\": [8, 8, 8]}"
    movement_policy_args: "{\\"score_threshold\\": %r}"
    segmentation_output_dir: "%s"
    inference_options { init_activation: 0.95 pad_value: 0.5 move_threshold: 0.6 segment_threshold: 0.6
                        min_boundary_dist { x: 2 y: 2 z: 1 } min_segment_size: 1500 disco_seed_threshold: %r }
  ''' % (vol_path, os.path.join(golden_dir, 'fib25_convstack.npz'), score, str(tmp_path / 'out'), disco_partial), req)
  runner = runner_mod.Runner(compute_mode=_lib.COMPUTE_FP16_TC)
  runner.start(req)
  try:
    assert runner.run((0, 0, 0), g64['volume'].shape) is not None
  finally:
    runner.stop_executor()
  seg, origins = storage.load_segmentation(str(tmp_path / 'out'), (0, 0, 0))

  hyb = _hybrid(engines['tc'], g64['volume'], seeds, opts)
  applied = np.asarray(hyb.disco_applied, dtype=bool)
  assert applied.any() and not applied.all()
  assert len(hyb.origins) >= 3
  np.testing.assert_array_equal(seg, np.maximum(hyb.segmentation, 0).astype(np.uint64))
  assert {k: (tuple(v.start_zyx), v.iters) for k, v in origins.items()} == \
      {k: (tuple(v[0]), v[1]) for k, v in hyb.origins.items()}


@pytest.mark.parametrize('name', ['disco_off', 'disco_never', 'disco_partial'])
def test_canvas_history_at_disco_thresholds(golden_dir, g64, engines, disco_partial, name):
  """ffn.inference.inference.Canvas(keep_history=True): history and history_deleted of one object equal the
  hybrid oracle's — no history_deleted at all when the disco merge is off."""
  from ffn.inference import executor, inference, inference_pb2, inference_utils
  from ffn.training.models import convstack_3d
  from ffn_b200 import _lib
  h = np.load(os.path.join(golden_dir, 'segment_at_history_64.npz'))
  start = tuple(int(v) for v in h['start'])
  opts = _options(name, disco_partial)
  model = convstack_3d.ConvStack3DFFNModel(fov_size=list(FOV), deltas=list(DELTAS), depth=12)
  exe = executor.B200Executor(executor.ExecutorInterface(), model, inference_utils.Counters(),
                              checkpoint_path=os.path.join(golden_dir, 'fib25_convstack.npz'),
                              compute_mode=_lib.COMPUTE_FP16_TC)
  try:
    req = inference_pb2.InferenceOptions(init_activation=0.95, pad_value=0.05, move_threshold=0.9,
                                         segment_threshold=0.6, min_segment_size=1000,
                                         disco_seed_threshold=opts.disco_seed_threshold)
    req.min_boundary_dist.x = req.min_boundary_dist.y = req.min_boundary_dist.z = 1
    cv = inference.Canvas(model.info, exe.get_client(inference_utils.Counters()), g64['volume'], req,
                          keep_history=True, image_mean=128, image_stddev=33)
    n = cv.segment_at(start)
    history, deleted = np.asarray(cv.history, np.int64).reshape(-1, 3), np.asarray(cv.history_deleted, np.int64)
  finally:
    exe.close()
  hyb = ff.Canvas(lambda s, im: engines['tc'].predict(s, im), _image(g64['volume']), FOV, DELTAS, opts)
  assert n == hyb.segment_at(start) > 5
  np.testing.assert_array_equal(history, np.asarray(hyb.history, np.int64).reshape(-1, 3))
  np.testing.assert_array_equal(deleted, np.asarray(hyb.history_deleted, np.int64))
  applied = np.asarray(hyb.disco_applied, dtype=bool)
  if name == 'disco_off':
    assert deleted.size == 0 and not applied.any()
  elif name == 'disco_never':
    assert deleted.size == n and not applied.any()
  else:
    assert deleted.size == n
