"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle and the golden
fixtures recorded from the reference's own Python modules.

Tolerances (also stated in DESIGN.md):
  * FFN_COMPUTE_FP32     logits max-abs <= 1e-4 vs the fp32 oracle; trajectories / labels identical to the
                         reference golden run; qprob within +-1 LSB.
  * FFN_COMPUTE_FP16X2_TC (fp16 hi+lo split operands on the tensor cores) logits max-abs <= 1e-4 vs the
                         fp32 oracle; trajectories / labels identical to the reference golden run — the
                         label-exact mode that runs on the tensor cores.
  * FFN_COMPUTE_FP16_TC  logits max-abs <= 4e-2 (fp16 operand rounding, fp32 accumulate; measured 3.1e-2) vs the
                         fp32 oracle and <= 1.5e-2 (measured 7.8e-3) vs the oracle with fp16-rounded conv
                         operands; flood-fill state BIT-EXACT vs the oracle
                         loop driven by the same GPU network ("hybrid oracle"): every integer / index /
                         decision is exact.  Against the pure fp32 reference golden the labels may differ
                         where a decision margin is below the logit error: label IoU after canonical
                         relabelling >= 0.97 on the golden volume (reported, see test_fp16_labels_vs_fp32_reference).
"""

import json
import os

import numpy as np
import pytest

from oracle import flood_fill as ff

pytestmark = pytest.mark.gpu

FOV, DELTAS = (33, 33, 33), (8, 8, 8)


@pytest.fixture(scope='module')
def weights(golden_dir):
  from ffn_b200 import tf_checkpoint
  return tf_checkpoint.load_convstack_npz(os.path.join(golden_dir, 'fib25_convstack.npz'))


@pytest.fixture(scope='module')
def engines(weights):
  from ffn_b200 import _lib, engine as eng
  w, b = weights
  out = {'fp32': eng.Engine(w, b, FOV, DELTAS, compute_mode=_lib.COMPUTE_FP32),
         'tc': eng.Engine(w, b, FOV, DELTAS, compute_mode=_lib.COMPUTE_FP16_TC),
         'x2': eng.Engine(w, b, FOV, DELTAS, compute_mode=_lib.COMPUTE_FP16X2_TC)}
  yield out
  for e in out.values():
    e.close()


@pytest.fixture(scope='module')
def g64(golden_dir):
  return np.load(os.path.join(golden_dir, 'flood_fill_64.npz'))


def _image(vol):
  return (vol.astype(np.float32) - np.float32(128.0)) / np.float32(33.0)


def test_wgmma_descriptor_known_answer():
  """wgmma with the K-major / no-swizzle descriptors the conv kernel uses, incl. tap shifts."""
  from ffn_b200 import engine as eng
  out = eng.selftest(n_out=16)
  assert out[0] == 0.0 and out[1] == 0.0 and out[2] == 0.0, out   # exact: small-integer operands
  assert out[3] > 1.0, 'swapped LBO/SBO must NOT reproduce the product'


@pytest.mark.parametrize('mode,tol', [('fp32', 1e-4), ('x2', 1e-4), ('tc', 4e-2)])
def test_predict_matches_oracle(engines, golden_dir, mode, tol):
  pat = np.load(os.path.join(golden_dir, 'net_patches.npz'))
  e = engines[mode]
  got = e.predict(pat['seed'], pat['image'])
  assert np.isfinite(got).all()
  e32, e64 = float(np.abs(got - pat['logits_fp32']).max()), float(np.abs(got - pat['logits_fp64']).max())
  print('%s: max |logit - oracle| = %.3g (fp32 oracle), %.3g (fp64 oracle), median %.3g' % (
      mode, e32, e64, float(np.median(np.abs(got - pat['logits_fp64'])))))
  assert e32 <= tol and e64 <= tol
  one = e.predict(pat['seed'][3], pat['image'][3])
  np.testing.assert_array_equal(one, got[3])                          # batch == single, deterministic
  np.testing.assert_array_equal(e.predict(pat['seed'][3], pat['image'][3]), one)


def test_predict_is_linear_in_nothing_but_respects_seed_add(engines):
  """Size-independent property: logits - seed (the update) does not depend on a constant added to
  the seed only through the network input, i.e. predict(seed) - seed == update(seed)."""
  rng = np.random.RandomState(0)
  img = rng.randn(*FOV).astype(np.float32)
  seed = np.full(FOV, -2.9444, np.float32)
  e = engines['fp32']
  a = e.predict(seed, img)
  assert np.abs((a - seed) - (e.predict(seed, img) - seed)).max() == 0.0


def test_fp32_segment_at_matches_reference_golden(engines, golden_dir, g64):
  from ffn_b200 import _lib, engine as eng
  gat = np.load(os.path.join(golden_dir, 'segment_at_64.npz'))
  cv = eng.DeviceCanvas(engines['fp32'], g64['volume'], eng.make_options(), 128.0, 33.0)
  st = cv.segment_at(tuple(int(v) for v in gat['start']))
  assert st.iters == int(gat['iters']) and st.finished
  seed = cv.read(_lib.ARRAY_SEED)
  want = gat['seed_canvas']
  np.testing.assert_array_equal(np.isnan(seed), np.isnan(want))
  ok = ~np.isnan(want)
  assert np.abs(seed[ok] - want[ok]).max() < 1e-3
  queue, done, start = cv.policy_state()
  assert queue.shape[0] == gat['queue'].shape[0] and start == tuple(int(v) for v in gat['start'])
  trace_cells = {tuple(((p - gat['start'] + 4) // 8).tolist()) for p in gat['trace']}
  assert {tuple(d) for d in done.tolist()} == trace_cells            # quantised done-set == visited lattice cells
  cv.close()


def _check_segment_all(cv, origins, overlaps, ctr, g, exact_qprob):
  from ffn_b200 import _lib
  seg = cv.read(_lib.ARRAY_SEGMENTATION)
  np.testing.assert_array_equal(seg, g['segmentation'])
  qp = cv.read(_lib.ARRAY_QPROB).astype(int)
  diff = np.abs(qp - g['seg_prob'].astype(int))
  assert diff.max() <= (0 if exact_qprob else 1)
  assert (diff > 0).mean() < 1e-3
  got = np.array([[o.id] + list(o.start_zyx) + [o.iters] for o in origins], dtype=np.int64).reshape(-1, 5)
  np.testing.assert_array_equal(got, g['origins'])
  ov = sorted((o.id, o.other_id, o.count) for o in overlaps)
  want = sorted(zip(*g['overlaps'].tolist())) if g['overlaps'].size else []
  assert ov == [tuple(int(v) for v in t) for t in want]
  gc = json.loads(str(g['counters']))
  assert ctr.inference_calls == gc['inference-calls']
  assert ctr.segment_at_calls == gc['segment_at-loop-calls']
  assert ctr.skip_threshold == gc.get('skip_threshold', 0)
  assert ctr.skip_invalid_pos == gc.get('skip_invalid_pos', 0)
  assert ctr.voxels_segmented == gc['voxels-segmented']
  assert ctr.voxels_overlapping == gc['voxels-overlapping']
  for sid, z, y, x, _ in g['origins']:
    assert seg[z, y, x] == sid                                       # every origin carries its own id


def test_fp16_logits_vs_fp16_operand_oracle(engines, weights, golden_dir):
  """The fp16 tensor-core path against the oracle with the SAME operand rounding (conv inputs and
  weights rounded to fp16, fp32 accumulate).  What is left is accumulation order — which still flips
  individual fp16 roundings of the next layer's operands (1 ulp = 5e-4 relative), so two correct fp16-operand
  implementations differ by a fraction of the rounding noise itself: measured 7.8e-3 here against 3.1e-2
  versus the fp32 oracle.  A kernel error (wrong tap, wrong halo) is O(1)."""
  from oracle.network import ConvStackOracle
  w, b = weights
  pat = np.load(os.path.join(golden_dir, 'net_patches.npz'))
  got = engines['tc'].predict(pat['seed'], pat['image'])
  want16 = ConvStackOracle(w, b, operand_round='fp16')(pat['seed'], pat['image'])
  err16 = float(np.abs(got - want16).max())
  err32 = float(np.abs(got - pat['logits_fp32']).max())
  print('fp16 TC: max |logit - fp16-operand oracle| = %.3g, vs fp32 oracle = %.3g' % (err16, err32))
  assert err16 <= 1.5e-2, err16
  assert err32 <= 4e-2, err32


def test_fp16_labels_vs_fp32_reference(engines, g64):
  """The fast fp16 mode against the PURE fp32 reference golden (not the hybrid oracle): fp16 operand
  rounding can move knife-edge decisions, so equality is not the claim — the label overlap is."""
  from ffn_b200 import _lib, engine as eng
  cv = eng.DeviceCanvas(engines['tc'], g64['volume'], eng.make_options(), 128.0, 33.0)
  origins, _, ctr = cv.segment_all(g64['seeds'])
  seg = cv.read(_lib.ARRAY_SEGMENTATION)
  cv.close()
  a = ff.canonical_relabel(np.maximum(seg, 0))
  b = ff.canonical_relabel(np.maximum(g64['segmentation'], 0))
  fg = (a > 0) | (b > 0)
  iou = float(((a == b) & fg).sum()) / float(fg.sum())
  mism = int((a != b).sum())
  steps_ref = int(json.loads(str(g64['counters']))['inference-calls'])
  print('fp16 TC vs fp32 reference golden: label IoU %.4f, %d mismatching voxels (%.2f%%), steps %d vs %d, '
        'segments %d vs %d' % (iou, mism, 100.0 * mism / a.size, ctr.inference_calls, steps_ref, len(origins),
                               g64['origins'].shape[0]))
  assert iou >= 0.97, iou
  assert len(origins) == g64['origins'].shape[0]
  assert abs(ctr.inference_calls - steps_ref) <= 0.05 * steps_ref


@pytest.mark.parametrize('mode', ['fp32', 'x2'])
def test_fp32_segment_all_matches_reference_golden(engines, g64, mode):
  """Whole-canvas run == the reference's Canvas.segment_all on the same volume / seeds / weights, in the
  fp32 CUDA-core mode AND in the split-fp16 tensor-core mode (label-exact on the tensor cores)."""
  from ffn_b200 import engine as eng
  cv = eng.DeviceCanvas(engines[mode], g64['volume'], eng.make_options(), 128.0, 33.0)
  origins, overlaps, ctr = cv.segment_all(g64['seeds'])
  _check_segment_all(cv, origins, overlaps, ctr, g64, exact_qprob=False)
  # idempotence: a second pass over the same seeds finds nothing new to segment
  seg_before = cv.read(1)
  o2, _, c2 = cv.segment_all(g64['seeds'])
  assert not o2 and c2.segments == ctr.segments
  np.testing.assert_array_equal((cv.read(1) > 0), (seg_before > 0))
  cv.close()


@pytest.mark.parametrize('mode', ['tc', 'fp32'])
def test_device_loop_bit_exact_vs_hybrid_oracle(engines, g64, mode):
  """Same network (the GPU's) under both loops: the reference loop restated on the CPU and the
  persistent kernel must agree bit for bit on seed, labels, qprob, origins, overlaps."""
  from ffn_b200 import _lib, engine as eng
  e = engines[mode]
  vol = g64['volume']
  cv = eng.DeviceCanvas(e, vol, eng.make_options(), 128.0, 33.0)
  origins, overlaps, ctr = cv.segment_all(g64['seeds'])
  hyb = ff.Canvas(lambda s, im: e.predict(s, im), _image(vol), FOV, DELTAS, ff.Options())
  hyb.segment_all(g64['seeds'])
  np.testing.assert_array_equal(cv.read(_lib.ARRAY_SEGMENTATION), hyb.segmentation)
  np.testing.assert_array_equal(cv.read(_lib.ARRAY_SEED), hyb.seed)
  qd = np.abs(cv.read(_lib.ARRAY_QPROB).astype(int) - hyb.seg_prob.astype(int))
  assert qd.max() <= 1 and (qd > 0).mean() < 1e-3                    # expf vs scipy expit at bin edges
  assert ctr.inference_calls == len(hyb.trace)
  assert [(o.id, tuple(o.start_zyx), o.iters) for o in origins] == \
      [(k, v[0], v[1]) for k, v in sorted(hyb.origins.items())]
  for k, v in hyb.overlaps.items():
    mine = sorted((o.other_id, o.count) for o in overlaps if o.id == k)
    assert mine == sorted(zip(v[0].tolist(), v[1].tolist()))
  assert ctr.skip_threshold == hyb.counters['skip_threshold']
  assert ctr.skip_invalid_pos == hyb.counters['skip_invalid_pos']
  cv.close()


def _run_segment_all(e, vol, seeds, chains, **opts):
  from ffn_b200 import _lib, engine as eng
  e.set_chains(chains)
  cv = eng.DeviceCanvas(e, vol, eng.make_options(**opts), 128.0, 33.0)
  origins, overlaps, ctr = cv.segment_all(seeds)
  out = dict(seg=cv.read(_lib.ARRAY_SEGMENTATION), seed=cv.read(_lib.ARRAY_SEED), qprob=cv.read(_lib.ARRAY_QPROB),
             origins=[(o.id, tuple(o.start_zyx), o.iters) for o in origins],
             overlaps=sorted((o.id, o.other_id, o.count) for o in overlaps),
             ctr={n: getattr(ctr, n) for n, _ in ctr._fields_ if n not in ('device_seconds', 'kernel_launches')},
             spec=cv.spec_stats())
  cv.close()
  e.set_chains(0)
  return out


@pytest.mark.parametrize('case', ['golden64', 'phantom'])
def test_chains_commit_in_seed_order(engines, g64, case):
  """Several objects in flight (chains, started ahead of their turn in private seed arrays) must give the
  results of the strictly sequential loop: labels, ids, origins (incl. per-object iters), overlaps, every
  counter, the probability map and Canvas.seed — bit for bit, because labels are committed in seed order and
  an early run that could have seen a different `segmentation > 0` answer is redone in turn."""
  from ffn_b200.synthetic import voronoi_phantom
  e = engines['tc']
  if case == 'golden64':
    vol, seeds, opts = g64['volume'], g64['seeds'], {}
  else:
    vol = voronoi_phantom((96, 112, 128), seed=7, cell_volume=40000.0)
    seeds = ff.grid_seeds(vol.shape, step=12, offsets=(0, 6))
    opts = dict(min_segment_size=3000)
  one = _run_segment_all(e, vol, seeds, 1, **opts)
  assert one['spec']['early_runs'] == 0 and one['spec']['steps_executed'] == one['ctr']['inference_calls']
  for chains in (2, 3, 4):
    many = _run_segment_all(e, vol, seeds, chains, **opts)
    print('%s, %d chains: %d early runs, %d discarded (%d steps), %d steps executed for %d counted' % (
        case, chains, many['spec']['early_runs'], many['spec']['early_runs_discarded'], many['spec']['steps_discarded'],
        many['spec']['steps_executed'], many['ctr']['inference_calls']))
    np.testing.assert_array_equal(many['seg'], one['seg'])
    np.testing.assert_array_equal(many['qprob'], one['qprob'])
    np.testing.assert_array_equal(many['seed'], one['seed'])
    assert many['origins'] == one['origins']
    assert many['overlaps'] == one['overlaps']
    assert many['ctr'] == one['ctr']
    assert many['spec']['steps_executed'] == many['ctr']['inference_calls'] + many['spec']['steps_discarded']
  assert len(one['origins']) >= 3


def test_batched_predict_shares_rounds(engines, golden_dir):
  """ffn_predict(batch): patches run four per round through one pipeline (executor.py:266-340 batches FoVs into
  one session.run); every patch's logits are bit-identical to its single-patch call, for any chain count."""
  pat = np.load(os.path.join(golden_dir, 'net_patches.npz'))
  e = engines['tc']
  seeds = np.concatenate([pat['seed'], pat['seed'][::-1], pat['seed'][:3]])
  imgs = np.concatenate([pat['image'], pat['image'][::-1], pat['image'][:3]])
  got = e.predict(seeds, imgs)                     # 13 patches: 3 full rounds + one of a single patch
  e.set_chains(1)
  ref = e.predict(seeds, imgs)
  np.testing.assert_array_equal(got, ref)
  for chains in (2, 3):
    e.set_chains(chains)
    np.testing.assert_array_equal(e.predict(seeds, imgs), ref)
  e.set_chains(0)
  for i in (0, 4, 12):
    np.testing.assert_array_equal(e.predict(seeds[i], imgs[i]), ref[i])


def test_device_movement_policy_known_answers(golden_dir):
  """get_scored_move_offsets + FaceMaxMovementPolicy.update on the DEVICE against the reference's own outputs
  (tests/golden/moves.npz: random faces, exact ties, nothing above threshold, anisotropic deltas).  A network
  with all-zero weights returns logits == the seed patch, so the canvas is loaded with the fixture's logits,
  ONE FoV step is run with the seed kept (reset_seed_per_segment=False) and the pushes are read from the
  event log: same offsets in the same order (descending (score, (dz, dy, dx)), movement.py:218)."""
  from ffn_b200 import _lib, engine as eng
  g = np.load(os.path.join(golden_dir, 'moves.npz'))
  th = float(g['threshold'])
  engines = {}
  checked = 0
  for i in range(int(g['n'])):
    logits = g['logits_%d' % i]
    deltas = tuple(int(v) for v in g['deltas_%d' % i])
    fov = tuple(int(v) for v in logits.shape)
    if min(fov) < 3:
      continue                                    # 2-D models are outside the engine's geometry
    key = (fov, deltas)
    if key not in engines:
      w = [np.zeros((3, 3, 3, 2 if l == 0 else 32, 32), np.float32) for l in range(4)] + [np.zeros((1, 1, 1, 32, 1), np.float32)]
      b = [np.zeros(32, np.float32) for _ in range(4)] + [np.zeros(1, np.float32)]
      engines[key] = eng.Engine(w, b, fov, deltas, compute_mode=_lib.COMPUTE_FP16_TC)
    e = engines[key]
    cv = eng.DeviceCanvas(e, np.zeros(fov, np.float32), eng.make_options(policy_score_threshold=th))
    pos = tuple(s // 2 for s in fov)
    seed = logits.astype(np.float32).copy()
    seed[pos] = np.float32(10.0)                  # the start voxel must pass is_valid_pos; it is on no face
    cv.write(_lib.ARRAY_SEED, seed)
    cv.start_trace(64)
    st = cv.segment_at(pos, max_steps=1, keep_seed=True)
    assert st.iters == 1
    ev = cv.get_trace()
    pushes = [tuple(int(v) - p for v, p in zip(r[1:4], pos)) for r in ev if r[0] == 1][1:]   # [0] is the start item
    moves = g['moves_%d' % i]
    want = sorted(((float(m[0]), (int(m[1]), int(m[2]), int(m[3]))) for m in moves), reverse=True)
    assert pushes == [w_[1] for w_ in want], (i, pushes, want)
    for off in pushes:                            # the score of a move is the logit at its position
      z, y, x = (p + o for p, o in zip(pos, off))
      assert float(logits[z, y, x]) >= th
    checked += 1
    cv.close()
  assert checked >= 20
  for e in engines.values():
    e.close()


def test_masks_and_rejections_vs_hybrid_oracle(engines):
  """Movement mask, seed mask, min_boundary_dist, small-object rejection (-1 markers)."""
  from ffn_b200 import _lib, engine as eng
  from ffn_b200.synthetic import voronoi_phantom
  e = engines['tc']
  vol = voronoi_phantom((56, 64, 72), seed=5, cell_volume=30000.0)
  mask = np.zeros(vol.shape, bool)
  mask[:, 30:34, :] = True
  seed_mask = np.zeros(vol.shape, bool)
  seed_mask[:, :, :24] = True
  opts = ff.Options(min_segment_size=40000, min_boundary_dist=(2, 3, 1))
  seeds = ff.grid_seeds(vol.shape, step=8, offsets=(0, 4))
  cv = eng.DeviceCanvas(e, vol, eng.make_options(min_segment_size=40000, min_boundary_dist_zyx=(2, 3, 1)), 128.0, 33.0)
  cv.set_mask(_lib.MASK_MOVEMENT, mask)
  cv.set_mask(_lib.MASK_SEED, seed_mask)
  origins, _, ctr = cv.segment_all(seeds)
  hyb = ff.Canvas(lambda s, im: e.predict(s, im), _image(vol), FOV, DELTAS, opts, mask=mask, seed_mask=seed_mask)
  hyb.segment_all(seeds)
  seg = cv.read(_lib.ARRAY_SEGMENTATION)
  np.testing.assert_array_equal(seg, hyb.segmentation)
  assert (seg == -1).sum() == (hyb.segmentation == -1).sum() > 0     # rejected seeds are marked
  assert ctr.skip_restricted_pos == hyb.counters['skip_restriced_pos']
  assert ctr.invalid_small == hyb.counters['invalid-small']
  assert len(origins) == len(hyb.origins)
  cv.close()


def test_update_at_and_init_seed(engines, g64):
  from ffn_b200 import _lib, engine as eng
  e = engines['fp32']
  vol = g64['volume']
  cv = eng.DeviceCanvas(e, vol, eng.make_options(), 128.0, 33.0)
  pos = (24, 40, 36)
  cv.init_seed(pos)
  pred = cv.update_at(pos)
  hyb = ff.Canvas(lambda s, im: e.predict(s, im), _image(vol), FOV, DELTAS, ff.Options())
  hyb.init_seed(pos)
  want = hyb.update_at(pos)
  np.testing.assert_array_equal(pred, want)
  np.testing.assert_array_equal(cv.read(_lib.ARRAY_SEED), hyb.seed)
  # a second init_seed clears exactly what was touched
  cv.init_seed((30, 30, 30))
  s = cv.read(_lib.ARRAY_SEED)
  assert np.isfinite(s).sum() == 1 and s[30, 30, 30] == np.float32(eng.f32_logit(0.95))
  cv.close()


def test_u8_and_f32_images_are_equivalent(engines, g64):
  from ffn_b200 import _lib, engine as eng
  e = engines['fp32']
  vol = g64['volume']
  a = eng.DeviceCanvas(e, vol, eng.make_options(), 128.0, 33.0)
  b = eng.DeviceCanvas(e, _image(vol), eng.make_options())
  np.testing.assert_array_equal(a.read(_lib.ARRAY_IMAGE), _image(vol))   # device normalisation == runner.py:383-385
  sa, sb = a.segment_at((16, 48, 32)), b.segment_at((16, 48, 32))
  assert sa.iters == sb.iters
  np.testing.assert_array_equal(a.read(_lib.ARRAY_SEED), b.read(_lib.ARRAY_SEED))
  a.close()
  b.close()


def test_pause_resume_and_box_io(engines, g64):
  """max_steps pauses inside an object; resuming reproduces the uninterrupted run."""
  from ffn_b200 import _lib, engine as eng
  e = engines['tc']
  vol = g64['volume']
  ref = eng.DeviceCanvas(e, vol, eng.make_options(), 128.0, 33.0)
  full = ref.segment_at((16, 48, 32))
  cv = eng.DeviceCanvas(e, vol, eng.make_options(), 128.0, 33.0)
  part = cv.segment_at((16, 48, 32), max_steps=11)
  assert part.iters == 11 and not part.finished
  rest = cv.segment_at((16, 48, 32), reset=False)
  assert rest.finished and rest.iters == full.iters
  np.testing.assert_array_equal(cv.read(_lib.ARRAY_SEED), ref.read(_lib.ARRAY_SEED))
  box = cv.read(_lib.ARRAY_SEED, (3, 5, 7), (10, 11, 12))
  np.testing.assert_array_equal(box, ref.read(_lib.ARRAY_SEED)[3:13, 5:16, 7:19])
  patch = np.arange(24, dtype=np.int32).reshape(2, 3, 4)
  cv.write(_lib.ARRAY_SEGMENTATION, patch, (1, 2, 3))
  np.testing.assert_array_equal(cv.read(_lib.ARRAY_SEGMENTATION)[1:3, 2:5, 3:7], patch)
  ref.close()
  cv.close()


def test_anisotropic_model_vs_oracle(weights):
  """configs[4] geometry: fov zyx (17,33,33), deltas (4,8,8), depth 9 (first 9 modules of FIB-25)."""
  from ffn_b200 import _lib, engine as eng
  from ffn_b200.synthetic import interior_seed, voronoi_phantom
  from oracle.network import ConvStackOracle
  w, b = weights
  w9, b9 = w[:18] + [w[-1]], b[:18] + [b[-1]]
  fov, deltas = (17, 33, 33), (4, 8, 8)
  vol = voronoi_phantom((40, 72, 72), seed=4, sigma=(0.5, 1.0, 1.0), voxel_size_zyx=(2.0, 1.0, 1.0))
  oracle_net = ConvStackOracle(w9, b9)
  for mode, tol in ((_lib.COMPUTE_FP32, 1e-4), (_lib.COMPUTE_FP16X2_TC, 1e-4), (_lib.COMPUTE_FP16_TC, 4e-2)):
    e = eng.Engine(w9, b9, fov, deltas, compute_mode=mode)
    rng = np.random.RandomState(1)
    img = _image(vol)[4:21, 8:41, 10:43]
    seed = np.where(rng.rand(*fov) < 0.3, rng.randn(*fov) * 2, -2.9444).astype(np.float32)
    assert np.abs(e.predict(seed, img) - oracle_net(seed, img)).max() <= tol
    cv = eng.DeviceCanvas(e, vol, eng.make_options(), 128.0, 33.0)
    start = interior_seed(vol, (20, 36, 36), max_radius=8)
    st = cv.segment_at(start)
    hyb = ff.Canvas(lambda s, im: e.predict(s, im), _image(vol), fov, deltas, ff.Options())
    n = hyb.segment_at(start)
    assert st.iters == n and n >= 1
    np.testing.assert_array_equal(cv.read(_lib.ARRAY_SEED), hyb.seed)
    cv.close()
    e.close()


def test_full_size_properties_256(engines):
  """BASELINE configs[1] size: invariants that do not need the (slow) CPU oracle."""
  from ffn_b200 import _lib, engine as eng
  from ffn_b200.synthetic import interior_seed, voronoi_phantom
  e = engines['tc']
  vol = voronoi_phantom((256, 256, 256), seed=1)
  cv = eng.DeviceCanvas(e, vol, eng.make_options(), 128.0, 33.0)
  start = interior_seed(vol, (128, 128, 128))
  st = cv.segment_at(start)
  assert st.finished and st.iters > 5
  seed = cv.read(_lib.ARRAY_SEED)
  lo = np.array(st.min_pos) - 16
  hi = np.array(st.max_pos) + 17
  outside = np.ones(seed.shape, bool)
  outside[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = False
  assert np.isnan(seed[outside]).all()                                # untouched voxels stay NaN
  assert seed[start] >= eng.f32_logit(0.9)                            # the seed survived
  queue, done, s0 = cv.policy_state()
  assert queue.shape[0] == 0 and done.shape[0] == st.iters            # one lattice cell per step
  again = cv.segment_at(start)                                        # deterministic
  assert again.iters == st.iters
  np.testing.assert_array_equal(cv.read(_lib.ARRAY_SEED), seed)
  cv.close()


def test_runner_end_to_end(tmp_path, golden_dir, g64):
  """Reference entry-point surface: InferenceRequest -> Runner.start/run -> seg-*.npz / .prob."""
  from google.protobuf import text_format
  from ffn.inference import inference_pb2, runner as runner_mod, storage
  vol_path = str(tmp_path / 'vol.npy')
  np.save(vol_path, g64['volume'])
  req = inference_pb2.InferenceRequest()
  text_format.Parse('''
    image { hdf5: "%s:raw" }
    image_mean: 128 image_stddev: 33 seed_policy: "PolicyGrid3d"
    model_checkpoint_path: "%s"
    model_name: "convstack_3d.ConvStack3DFFNModel"
    model_args: "{\\"depth\\": 12, \\"fov_size\\": [33, 33, 33], \\"deltas\\": [8, 8, 8]}"
    segmentation_output_dir: "%s"
    inference_options { init_activation: 0.95 pad_value: 0.05 move_threshold: 0.9
                        min_boundary_dist { x: 1 y: 1 z: 1} segment_threshold: 0.6 min_segment_size: 1000 }
  ''' % (vol_path, os.path.join(golden_dir, 'fib25_convstack.npz'), str(tmp_path / 'out')), req)
  from ffn_b200 import _lib
  runner = runner_mod.Runner(compute_mode=_lib.COMPUTE_FP32)
  runner.start(req)
  canvas = runner.run((0, 0, 0), g64['volume'].shape)
  assert canvas is not None
  seg, origins = storage.load_segmentation(str(tmp_path / 'out'), (0, 0, 0))
  want = g64['segmentation'].copy()
  want[want < 0] = 0
  np.testing.assert_array_equal(seg, want.astype(np.uint64))
  assert sorted(origins) == g64['origins'][:, 0].tolist()
  assert origins[4].start_zyx == tuple(g64['origins'][3, 1:4]) and origins[4].iters == g64['origins'][3, 4]
  with np.load(storage.object_prob_path(str(tmp_path / 'out'), (0, 0, 0))) as z:
    assert np.abs(z['qprob'].astype(int) - g64['seg_prob'].astype(int)).max() <= 1
  assert canvas.counters['inference-calls'].value == g64['trace'].shape[0]
  assert runner.counters['voxels-segmented'].value == int((want > 0).sum())
  assert runner.run((0, 0, 0), g64['volume'].shape) is None          # idempotent restart (runner.py:509-510)
  runner.stop_executor()


def test_canvas_checkpoint_roundtrip(tmp_path, golden_dir, g64):
  """save_checkpoint / restore_checkpoint with an object in flight resumes to the same result."""
  from ffn.inference import executor, inference, inference_pb2, inference_utils, seed as seed_mod
  from ffn.training.models import convstack_3d
  from ffn_b200 import _lib
  model = convstack_3d.ConvStack3DFFNModel(fov_size=[33, 33, 33], deltas=[8, 8, 8], depth=12)
  exe = executor.B200Executor(executor.ExecutorInterface(), model, inference_utils.Counters(),
                              checkpoint_path=os.path.join(golden_dir, 'fib25_convstack.npz'),
                              compute_mode=_lib.COMPUTE_FP32)
  opts = inference_pb2.InferenceOptions(init_activation=0.95, pad_value=0.05, move_threshold=0.9,
                                        segment_threshold=0.6, min_segment_size=1000)
  opts.min_boundary_dist.x = opts.min_boundary_dist.y = opts.min_boundary_dist.z = 1

  def make():
    return inference.Canvas(model.info, exe.get_client(inference_utils.Counters()), g64['volume'], opts,
                            keep_probability_maps=True, image_mean=128, image_stddev=33)
  a = make()
  start = (16, 48, 32)
  n = a.segment_at(start, max_steps=20)
  assert n == 20
  path = str(tmp_path / 'c.cpoint')
  a.seed_policy = seed_mod.PolicyGrid3d(a)
  a.save_checkpoint(path, partial_segment_iters=n)
  b = make()
  partial = b.restore_checkpoint(path)
  assert partial == 20
  np.testing.assert_array_equal(np.asarray(b.seed), np.asarray(a.seed))
  total_b = b.segment_at(start, partial_segment_iters=partial)
  total_a = a.segment_at(start, partial_segment_iters=n)
  assert total_a == total_b == 80
  np.testing.assert_array_equal(np.asarray(b.seed), np.asarray(a.seed))
  exe.close()


def test_segment_all_resumes_mid_object_checkpoint(tmp_path, golden_dir, g64):
  """A checkpoint taken INSIDE an object (the reference saves the seed policy one step back, inference.py:745-747):
  restore + segment_all finishes that object and goes on with the NEXT seed — the in-flight seed is not run a
  second time — and the result equals the uninterrupted reference run."""
  from ffn.inference import executor, inference, inference_pb2, inference_utils, seed as seed_mod
  from ffn.training.models import convstack_3d
  from ffn_b200 import _lib
  model = convstack_3d.ConvStack3DFFNModel(fov_size=[33, 33, 33], deltas=[8, 8, 8], depth=12)
  exe = executor.B200Executor(executor.ExecutorInterface(), model, inference_utils.Counters(),
                              checkpoint_path=os.path.join(golden_dir, 'fib25_convstack.npz'),
                              compute_mode=_lib.COMPUTE_FP16X2_TC)
  opts = inference_pb2.InferenceOptions(init_activation=0.95, pad_value=0.05, move_threshold=0.9,
                                        segment_threshold=0.6, min_segment_size=1000)
  opts.min_boundary_dist.x = opts.min_boundary_dist.y = opts.min_boundary_dist.z = 1
  seeds = np.asarray(g64['seeds'])

  class ListPolicy(seed_mod.BaseSeedPolicy):
    def init_coords(self):
      self.coords = seeds.copy()

  def make():
    return inference.Canvas(model.info, exe.get_client(inference_utils.Counters()), g64['volume'], opts,
                            keep_probability_maps=True, image_mean=128, image_stddev=33)
  # an object of the golden run with enough steps to stop inside: the seeds in front of it are processed normally
  row = next(r for r in g64['origins'] if int(r[4]) >= 15)
  k = next(i for i, sd in enumerate(seeds.tolist()) if tuple(sd) == tuple(int(v) for v in row[1:4]))

  class HeadPolicy(seed_mod.BaseSeedPolicy):
    def init_coords(self):
      self.coords = seeds[:k].copy()
  a = make()
  a.segment_all(seed_policy=HeadPolicy)
  a.seed_policy = ListPolicy(a)
  a.seed_policy.init_coords()
  a.seed_policy.idx = k + 1                       # the policy has handed out seed k, which is now in flight
  n = a.segment_at(tuple(int(v) for v in seeds[k]), max_steps=7)
  assert n == 7
  path = str(tmp_path / 'mid.cpoint')
  a.save_checkpoint(path, partial_segment_iters=n)
  b = make()
  assert b.restore_checkpoint(path) == 7
  b.segment_all(seed_policy=ListPolicy)
  np.testing.assert_array_equal(np.asarray(b.segmentation), g64['segmentation'])
  assert sorted((v.start_zyx, v.iters) for v in b.origins.values()) == sorted(
      (tuple(int(x) for x in row[1:4]), int(row[4])) for row in g64['origins'])
  assert b.counters['segment_at-loop-calls'].value >= 1
  exe.close()


def test_concurrent_canvases_batch_size_two(golden_dir, g64):
  """InferenceRequest.batch_size semantics: two canvases served concurrently (two engines, half the
  SMs each, one host thread per canvas) produce exactly what the whole-GPU engine produces."""
  import threading
  from ffn.inference import executor, inference, inference_pb2, inference_utils, seed as seed_mod
  from ffn.training.models import convstack_3d
  from ffn_b200 import _lib
  model = convstack_3d.ConvStack3DFFNModel(fov_size=[33, 33, 33], deltas=[8, 8, 8], depth=12)
  opts = inference_pb2.InferenceOptions(init_activation=0.95, pad_value=0.05, move_threshold=0.9,
                                        segment_threshold=0.6, min_segment_size=1000)
  opts.min_boundary_dist.x = opts.min_boundary_dist.y = opts.min_boundary_dist.z = 1
  ckpt = os.path.join(golden_dir, 'fib25_convstack.npz')
  vols = [g64['volume'], np.ascontiguousarray(g64['volume'][::-1])]

  def run(exe, vol, out, i):
    cv = inference.Canvas(model.info, exe.get_client(inference_utils.Counters()), vol, opts,
                          keep_probability_maps=True, image_mean=128, image_stddev=33)
    cv.segment_all(seed_policy=seed_mod.PolicyGrid3d)
    out[i] = (np.asarray(cv.segmentation), np.asarray(cv.seg_prob), dict(cv.origins))

  ref_exe = executor.B200Executor(executor.ExecutorInterface(), model, inference_utils.Counters(), batch_size=1,
                                  checkpoint_path=ckpt)
  want = [None, None]
  for i in range(2):
    run(ref_exe, vols[i], want, i)
  ref_exe.close()

  exe = executor.B200Executor(executor.ExecutorInterface(), model, inference_utils.Counters(), batch_size=2,
                              checkpoint_path=ckpt)
  assert len(exe.engines) == 2 and exe.engines[0].info()['grid'] * 2 <= exe.engines[0].info()['sm_count']
  got = [None, None]
  threads = [threading.Thread(target=run, args=(exe, vols[i], got, i)) for i in range(2)]
  for t in threads:
    t.start()
  for t in threads:
    t.join()
  exe.close()
  for i in range(2):
    np.testing.assert_array_equal(got[i][0], want[i][0])
    np.testing.assert_array_equal(got[i][1], want[i][1])
    assert {k: (v.start_zyx, v.iters) for k, v in got[i][2].items()} == \
        {k: (v.start_zyx, v.iters) for k, v in want[i][2].items()}


class _HostCanvas:
  """Just enough canvas for the host (scipy) PolicyPeaks path: no `_dev`."""

  def __init__(self, image, segmentation, restrictor, voxel_size_zyx, margin):
    self.image, self.segmentation, self.restrictor = image, segmentation, restrictor
    self.voxel_size_zyx, self.margin, self.shape = voxel_size_zyx, margin, image.shape


@pytest.mark.parametrize('voxel', [(1, 1, 1), (2, 1, 1)])
def test_device_policy_peaks_equals_oracle(golden_dir, voxel):
  """PolicyPeaks on the device (Sobel, adaptive threshold, exact EDT, peak picking) against the oracle's
  independent restatement (oracle/seed_peaks.py: scipy Sobel / gaussian / exact EDT pinned to the O(n^2)
  definition, documented peak_local_max semantics): the SAME coordinates in the SAME order, with masks, an
  already-segmented region and anisotropic voxels (ffn/inference/seed.py:133-199)."""
  from ffn.inference import executor, inference, inference_pb2, inference_utils, movement, seed as seed_mod
  from ffn.training.models import convstack_3d
  from ffn_b200 import synthetic
  from oracle import seed_peaks
  model = convstack_3d.ConvStack3DFFNModel(fov_size=[33, 33, 33], deltas=[8, 8, 8], depth=12)
  exe = executor.B200Executor(executor.ExecutorInterface(), model, inference_utils.Counters(),
                              checkpoint_path=os.path.join(golden_dir, 'fib25_convstack.npz'))
  opts = inference_pb2.InferenceOptions(init_activation=0.95, pad_value=0.05, move_threshold=0.9,
                                        segment_threshold=0.6, min_segment_size=1000)
  shape = (72, 90, 101)
  vol = synthetic.voronoi_phantom(shape, seed=5, cell_volume=12000.0)
  rng = np.random.RandomState(3)
  mask = np.zeros(shape, dtype=bool)
  mask[:, :12, :] = True
  seed_mask = rng.rand(*shape) > 0.995
  restrictor = movement.MovementRestrictor(mask=mask, seed_mask=seed_mask)
  cv = inference.Canvas(model.info, exe.get_client(inference_utils.Counters()), vol, opts, restrictor=restrictor,
                        voxel_size_zyx=voxel, image_mean=128, image_stddev=33)
  seg = np.zeros(shape, dtype=np.int32)
  seg[40:60, 50:80, 20:70] = 7
  cv.segmentation[...] = seg
  got = seed_mod.PolicyPeaks(cv).remaining()

  image = (vol.astype(np.float32) - np.float32(128)) / np.float32(33)
  want = seed_peaks.policy_peaks(image, voxel_size_zyx=voxel, segmentation=seg, mask=mask, seed_mask=seed_mask,
                                 margin_zyx=cv.margin)
  assert want.shape[0] > 20
  a = set(map(tuple, got.tolist()))
  b = set(map(tuple, want.tolist()))
  print('PolicyPeaks voxel %r: device %d seeds, oracle %d, common %d; only device %r; only oracle %r' % (
      voxel, len(a), len(b), len(a & b), sorted(a - b)[:5], sorted(b - a)[:5]))
  np.testing.assert_array_equal(got, want)
  assert not any(mask[z, y, x] or seed_mask[z, y, x] or seg[z, y, x] > 0 for z, y, x in got)
  exe.close()


def test_keep_history_matches_reference_golden(golden_dir, g64):
  """Canvas(keep_history=True): history (positions visited) and history_deleted (per step, voxels whose
  old seed >= logit(0.8) got a raw logit < 0) equal the reference's own run (inference.py:420-422,
  :520-521; fixture from tests/golden/make_golden_history.py), in the label-exact fp32 mode."""
  from ffn.inference import executor, inference, inference_pb2, inference_utils
  from ffn.training.models import convstack_3d
  from ffn_b200 import _lib
  h = np.load(os.path.join(golden_dir, 'segment_at_history_64.npz'))
  model = convstack_3d.ConvStack3DFFNModel(fov_size=[33, 33, 33], deltas=[8, 8, 8], depth=12)
  exe = executor.B200Executor(executor.ExecutorInterface(), model, inference_utils.Counters(),
                              checkpoint_path=os.path.join(golden_dir, 'fib25_convstack.npz'),
                              compute_mode=_lib.COMPUTE_FP32)
  opts = inference_pb2.InferenceOptions(init_activation=0.95, pad_value=0.05, move_threshold=0.9,
                                        segment_threshold=0.6, min_segment_size=1000)
  opts.min_boundary_dist.x = opts.min_boundary_dist.y = opts.min_boundary_dist.z = 1
  cv = inference.Canvas(model.info, exe.get_client(inference_utils.Counters()), g64['volume'], opts,
                        keep_history=True, image_mean=128, image_stddev=33)
  n = cv.segment_at(tuple(int(v) for v in h['start']))
  assert n == h['history'].shape[0]
  np.testing.assert_array_equal(np.asarray(cv.history, np.int32).reshape(-1, 3), h['history'])
  np.testing.assert_array_equal(np.asarray(cv.history_deleted, np.int64), h['history_deleted'])
  cv.segment_at(tuple(int(v) for v in h['second_start']))
  np.testing.assert_array_equal(np.asarray(cv.history, np.int32).reshape(-1, 3), h['second_history'])
  np.testing.assert_array_equal(np.asarray(cv.history_deleted, np.int64), h['second_history_deleted'])
  exe.close()


def test_resegmentation_process_point(tmp_path, golden_dir):
  """resegmentation.process_point (resegmentation.py:114-293) through Runner + the device canvas with
  keep_history: a pair point between two ground-truth cells and an endpoint; the re-grown objects recover
  the cells they were seeded in, histories / deletes have one entry per FoV step."""
  from google.protobuf import text_format
  from ffn.inference import inference_pb2, resegmentation, runner as runner_mod
  from ffn_b200 import synthetic
  shape = (96, 96, 96)
  vol, cells = synthetic.voronoi_phantom(shape, seed=7, cell_volume=45000.0, return_cells=True)
  np.save(tmp_path / 'vol.npy', vol)
  np.save(tmp_path / 'seg.npy', cells[np.newaxis].astype(np.uint64))
  # a decision point: a membrane voxel (label 0) near the centre with different cells on its -x / +x side
  c = 48
  found = None
  for z in range(c - 8, c + 9):
    for y in range(c - 8, c + 9):
      for x in range(c - 8, c + 9):
        if cells[z, y, x] != 0 or found is not None:
          continue
        left = [int(v) for v in cells[z, y, x - 4:x][::-1] if v > 0]
        right = [int(v) for v in cells[z, y, x + 1:x + 5] if v > 0]
        if left and right and left[0] != right[0]:
          found = (z, y, x, left[0], right[0])
  assert found is not None
  z, y, x, id_a, id_b = found
  req = inference_pb2.ResegmentationRequest()
  text_format.Parse('''inference { image { hdf5: "%s:raw" } init_segmentation { hdf5: "%s:seg" }
      image_mean: 128 image_stddev: 33 seed_policy: "PolicyPeaks" model_checkpoint_path: "%s"
      model_name: "convstack_3d.ConvStack3DFFNModel"
      model_args: "{\\"depth\\": 12, \\"fov_size\\": [33, 33, 33], \\"deltas\\": [8, 8, 8]}"
      segmentation_output_dir: "%s"
      inference_options { init_activation: 0.95 pad_value: 0.05 move_threshold: 0.9 min_boundary_dist { x: 1 y: 1 z: 1}
                          segment_threshold: 0.6 min_segment_size: 1000 } }
      radius { x: 40 y: 40 z: 40 } output_directory: "%s" max_retry_iters: 2
      exclusion_radius { x: 4 y: 4 z: 4 } analysis_radius { x: 24 y: 24 z: 24 }''' % (
          tmp_path / 'vol.npy', tmp_path / 'seg.npy', os.path.join(golden_dir, 'fib25_convstack.npz'),
          tmp_path / 'segout', tmp_path / 'reseg'), req)
  for ids in ((id_a, id_b), (id_a,)):
    pt = req.points.add()
    pt.id_a = ids[0]
    if len(ids) > 1:
      pt.id_b = ids[1]
    pt.point.x, pt.point.y, pt.point.z = x, y, z
  runner = runner_mod.Runner()
  runner.start(req.inference)
  resegmentation.process(req, runner)
  runner.stop_executor()

  sub = cells[z - 40:z + 41, y - 40:y + 41, x - 40:x + 41]
  for n, ids in enumerate(((id_a, id_b), (id_a,))):
    path = resegmentation.get_target_path(req, n)
    assert path is None                                                  # i.e. the result exists
    name = '%d-%d_at_%d_%d_%d.npz' % (ids[0], ids[1] if len(ids) > 1 else 0, x, y, z)
    out = np.load(tmp_path / 'reseg' / name, allow_pickle=True)
    assert out['probs'].shape == (len(ids), 81, 81, 81) and out['raw_probs'].dtype == np.uint8
    assert tuple(out['corner_zyx']) == (z - 40, y - 40, x - 40) and not bool(out['is_shift'])
    assert inference_pb2.ResegmentationRequest.FromString(out['request'].tobytes() if hasattr(out['request'], 'tobytes')
                                                           else bytes(out['request'])).radius.x == 40
    for k, sid in enumerate(ids):
      hist, dele, starts = out['histories'][k], out['deletes'][k], out['start_points'][k]
      assert len(starts) >= 1 and len(hist) == len(dele) and len(hist) > 3
      grown = out['raw_probs'][k] >= 154                                 # quantised 0.6
      orig = sub == sid
      # the object re-grown from inside cell `sid` recovers most of it and stays mostly inside it
      assert (grown & orig).sum() > 0.3 * orig.sum(), ((grown & orig).sum(), orig.sum())
      assert (grown & orig).sum() > 0.7 * grown.sum(), ((grown & orig).sum(), grown.sum())


@pytest.mark.parametrize('mode', ['fp32', 'x2'])
def test_resegmentation_process_point_equals_reference_golden(tmp_path, golden_dir, g64, mode):
  """resegmentation.process_point against the REFERENCE's own process_point (resegmentation.py:111-293, run unmodified by
  tests/golden/make_golden_reseg.py with the fp32 oracle network) on the golden volume: a pair point between two
  objects of the reference's own segmentation and the same point as an endpoint.  Seeding (EDT maximum, margins,
  init_exclusion_radius), the attempts, histories, history_deleted, the recovery test inside the analysis window and
  the saved arrays must be the reference's — in both label-exact modes."""
  from google.protobuf import text_format
  from ffn.inference import inference_pb2, resegmentation, runner as runner_mod
  from ffn_b200 import _lib
  r = np.load(os.path.join(golden_dir, 'reseg_64.npz'))
  pz, py, px = (int(v) for v in r['point_zyx'])
  id_a, id_b = int(r['id_a']), int(r['id_b'])
  rz, ry, rx = (int(v) for v in r['radius_zyx'])
  az, ay, ax = (int(v) for v in r['analysis_radius_zyx'])
  np.save(tmp_path / 'vol.npy', g64['volume'])
  np.save(tmp_path / 'seg.npy', np.maximum(g64['segmentation'], 0)[np.newaxis].astype(np.uint64))
  req = inference_pb2.ResegmentationRequest()
  text_format.Parse('''inference { image { hdf5: "%s:raw" } init_segmentation { hdf5: "%s:seg" }
      image_mean: 128 image_stddev: 33 seed_policy: "PolicyPeaks" model_checkpoint_path: "%s"
      model_name: "convstack_3d.ConvStack3DFFNModel"
      model_args: "{\\"depth\\": 12, \\"fov_size\\": [33, 33, 33], \\"deltas\\": [8, 8, 8]}"
      segmentation_output_dir: "%s"
      inference_options { init_activation: 0.95 pad_value: 0.05 move_threshold: 0.9 min_boundary_dist { x: 1 y: 1 z: 1}
                          segment_threshold: 0.6 min_segment_size: 1000 } }
      radius { x: %d y: %d z: %d } output_directory: "%s" max_retry_iters: %d
      exclusion_radius { x: %d y: %d z: %d } init_exclusion_radius { x: %d y: %d z: %d }
      analysis_radius { x: %d y: %d z: %d } segment_recovery_fraction: %r''' % (
          tmp_path / 'vol.npy', tmp_path / 'seg.npy', os.path.join(golden_dir, 'fib25_convstack.npz'),
          tmp_path / 'segout', rx, ry, rz, tmp_path / 'reseg', int(r['max_retry_iters']),
          *([int(r['exclusion_radius'])] * 3), *([int(r['init_exclusion_radius'])] * 3), ax, ay, az,
          float(r['segment_recovery_fraction'])), req)
  for ids in ((id_a, id_b), (id_a,)):
    pt = req.points.add()
    pt.id_a = ids[0]
    if len(ids) > 1:
      pt.id_b = ids[1]
    pt.point.x, pt.point.y, pt.point.z = px, py, pz
  runner = runner_mod.Runner(compute_mode={'fp32': _lib.COMPUTE_FP32, 'x2': _lib.COMPUTE_FP16X2_TC}[mode])
  runner.start(req.inference)
  resegmentation.process(req, runner)
  runner.stop_executor()
  for tag, ids in (('pair', (id_a, id_b)), ('endpoint', (id_a,))):
    name = '%d-%d_at_%d_%d_%d.npz' % (ids[0], ids[1] if len(ids) > 1 else 0, px, py, pz)
    out = np.load(tmp_path / 'reseg' / name, allow_pickle=True)
    np.testing.assert_array_equal(np.asarray(out['corner_zyx']), r[tag + '_corner_zyx'])
    assert bool(out['is_shift']) == bool(r[tag + '_is_shift'])
    n_obj = int(r[tag + '_n_objects'])
    assert len(out['histories']) == n_obj and len(out['deletes']) == n_obj
    for k in range(2):
      np.testing.assert_array_equal(np.asarray(out['start_points'][k], dtype=np.int64).reshape(-1, 3), r['%s_starts_%d' % (tag, k)])
    for k in range(n_obj):
      np.testing.assert_array_equal(np.asarray(out['histories'][k], dtype=np.int32).reshape(-1, 3), r['%s_history_%d' % (tag, k)])
      np.testing.assert_array_equal(np.asarray(out['deletes'][k], dtype=np.int64), r['%s_deletes_%d' % (tag, k)])
    for key in ('raw_probs', 'probs'):
      got, want = out[key].astype(int), r['%s_%s' % (tag, key)].astype(int)
      assert got.shape == want.shape
      diff = np.abs(got - want)
      assert diff.max() <= 1 and (diff > 0).mean() < 1e-3, (key, int(diff.max()), float((diff > 0).mean()))   # quantisation bin edges


def test_configs1_object_vs_pure_fp32_oracle(engines, weights):
  """BASELINE configs[1] (256^3 phantom seed 1, one object from the centre; run on the 144^3 neighbourhood of the seed
  so that the CPU side stays small) against the PURE fp32 oracle on the CPU (reference loop + fp32 network, no device
  arithmetic in the checker), the whole object (a few hundred FoV steps): the split-fp16 mode must walk the same
  positions and leave the same seed canvas unless a decision sits on a knife edge (then the object must still agree
  voxel for voxel to 99 %); the fast fp16 mode is bounded by the overlap of the object it grows."""
  import torch
  from ffn_b200 import _lib, engine as eng
  from ffn_b200.synthetic import interior_seed, voronoi_phantom
  from oracle.network import ConvStackOracle
  vol = voronoi_phantom((256, 256, 256), seed=1)
  start = interior_seed(vol, (128, 128, 128))
  # the object stays inside its cell: a crop around it keeps the oracle's arrays small; positions are crop-relative
  lo = np.array(start) - 72
  crop = vol[lo[0]:lo[0] + 144, lo[1]:lo[1] + 144, lo[2]:lo[2] + 144]
  cstart = tuple(int(v) for v in np.array(start) - lo)
  torch.set_num_threads(min(32, os.cpu_count() or 1))
  w, b = weights
  orc = ff.Canvas(ConvStackOracle(w, b), _image(crop), FOV, DELTAS, ff.Options())
  n_ref = orc.segment_at(cstart)
  ref_mask = orc.seed >= ff.f32_logit(0.6)
  assert n_ref > 50 and ref_mask.sum() > 10000
  th = eng.f32_logit(0.6)
  report = {}
  for mode in ('x2', 'tc'):
    cv = eng.DeviceCanvas(engines[mode], crop, eng.make_options(), 128.0, 33.0)
    cv.start_trace(1 << 16)
    st = cv.segment_at(cstart)
    ev = cv.get_trace()
    steps = ev[ev[:, 0] == 6][:, 1:]
    seed = cv.read(_lib.ARRAY_SEED)
    cv.close()
    mask = seed >= th
    iou = float((mask & ref_mask).sum()) / float((mask | ref_mask).sum())
    same = int(st.iters) == n_ref and np.array_equal(steps, np.asarray(orc.trace, dtype=steps.dtype).reshape(-1, 3))
    n_same = 0
    for a, b2 in zip(steps.tolist(), [list(p) for p in orc.trace]):
      if a != b2:
        break
      n_same += 1
    both = np.isfinite(seed) & np.isfinite(orc.seed)
    err = float(np.abs(seed[both] - orc.seed[both]).max()) if same else float('nan')
    report[mode] = dict(steps=int(st.iters), steps_ref=n_ref, same_positions=bool(same), first_divergent_step=n_same,
                        object_iou=round(iou, 5), max_seed_err=err, min_margin_ref=float(orc.min_margin))
    if mode == 'x2':
      assert (same and err <= 1e-3) or iou >= 0.99, report
    else:
      assert iou >= 0.95 and abs(int(st.iters) - n_ref) <= 0.15 * n_ref, report
  print('configs[1] object vs pure fp32 oracle:', json.dumps(report))

