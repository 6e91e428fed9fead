"""The conv stack and the flood fill pinned bit for bit with exactly representable networks (oracle/exact_net.py).

Under the premise that tests/test_exact_net.py checks on the CPU for every network and input used here, every correct
implementation computes the same logits, so the device must equal the float64 oracle with assert_array_equal, no
tolerance: the fp32 and split-fp16 modes the plain oracle, the fp16 tensor-core mode the fp16-operand oracle.

a. ffn_predict at every case of EXACT_SWEEP (the geometries of tests/test_geometry_oracle.py:SWEEP, and depths 1, 2, 12
   and 16), batches of 1, 4, 5 and 9 patches, on the default grid and on 7 CTAs, with 1 and 4 chains.
b. Every probe network (fp32-only residual, biases and seeds, fp16 rounding ties, subnormal operands, ReLU at zero and
   the order of the last sum) in all three modes.
c. The profiled build (enable_profiling) gives the plain build's logits and flood fill bit for bit, with sane
   counters.
d. segment_all with the flood network on a u8 canvas in all three modes with 1 and 4 chains: labels, seed canvas,
   origins, overlaps and counters equal the pure CPU oracle loop and the reference's own run
   (tests/golden/exact_flood_fill.npz); one segment_at.
e. The flagship geometry (33, 33, 33) / depth 12: the device loop equals the hybrid oracle, and some of the patches
   it fed the network are checked against the float64 oracle.
"""

import json
import os

import numpy as np
import pytest

from oracle import exact_net as xn
from oracle import flood_fill as ff
from test_exact_net import EXACT_SWEEP, PROBE_FOV, flood_case, sweep_case

pytestmark = pytest.mark.gpu


def _modes():
  from ffn_b200 import _lib
  return {'tc': (_lib.COMPUTE_FP16_TC, 'fp16'), 'x2': (_lib.COMPUTE_FP16X2_TC, 'x2'), 'fp32': (_lib.COMPUTE_FP32, 'fp32')}


def _deltas(fov):
  return tuple(min(8, f // 2) for f in fov)


def _want(w, b, seeds, imgs, omode):
  return xn.logits(w, b, seeds, imgs, 'fp16' if omode == 'fp16' else 'fp32')


def _assert_equal(got, want, what):
  if not np.array_equal(got, want):
    d = np.abs(got.astype(np.float64) - want.astype(np.float64))
    i = np.unravel_index(int(np.argmax(d)), d.shape)
    pytest.fail('%s: %d of %d logits differ, max |diff| %.3g at %r (got %r, want %r)' % (
        what, int((got != want).sum()), got.size, d.max(), i, float(got[i]), float(want[i])))


@pytest.mark.parametrize('case', [c[0] for c in EXACT_SWEEP])
def test_predict_equals_the_oracle_exactly(case):
  from ffn_b200 import engine as eng
  fov, depth, w, b, seeds, imgs = sweep_case(case)
  n = seeds.shape[0]
  for name, (mode, omode) in _modes().items():
    want = _want(w, b, seeds, imgs, omode)
    e = eng.Engine(w, b, fov, _deltas(fov), compute_mode=mode)
    for grid in (0, min(7, e.info()['tiles'])):
      e.set_grid(grid)
      for chains in (1, 4):
        e.set_chains(chains)
        for k in sorted({1, n} | {m for m in (4, 5, 9) if m <= n}):
          got = e.predict(seeds[:k], imgs[:k])
          _assert_equal(got, want[:k], '%s %s grid %d chains %d batch %d' % (case, name, grid, chains, k))
    e.close()


@pytest.mark.parametrize('name', sorted(xn.PROBES))
def test_probe_equals_the_oracle_exactly(name):
  from ffn_b200 import engine as eng
  w, b, seeds, imgs = xn.PROBES[name](PROBE_FOV)
  for mname, (mode, omode) in _modes().items():
    e = eng.Engine(w, b, PROBE_FOV, _deltas(PROBE_FOV), compute_mode=mode)
    _assert_equal(e.predict(seeds, imgs), _want(w, b, seeds, imgs, omode), '%s %s' % (name, mname))
    e.close()


def _flood(e, vol, seeds, opts):
  """segment_all on a fresh device canvas: the state every flood test compares."""
  from ffn_b200 import _lib, engine as eng
  o = dict(opts)
  cv = eng.DeviceCanvas(e, vol, eng.make_options(min_boundary_dist_zyx=o.pop('min_boundary_dist'), **o),
                        xn.FLOOD_MEAN, xn.FLOOD_STDDEV)
  origins, overlaps, ctr = cv.segment_all(seeds)
  out = dict(seg=cv.read(_lib.ARRAY_SEGMENTATION), seed=cv.read(_lib.ARRAY_SEED), qprob=cv.read(_lib.ARRAY_QPROB),
             origins=[(o.id, tuple(int(v) for v in o.start_zyx), o.iters) for o in origins],
             overlaps=sorted((o.id, o.other_id, o.count) for o in overlaps), ctr=ctr)
  cv.close()
  return out


def _check_flood(dev, cpu, what):
  np.testing.assert_array_equal(dev['seg'], cpu.segmentation, err_msg=what)
  np.testing.assert_array_equal(dev['seed'], cpu.seed, err_msg=what)
  qd = np.abs(dev['qprob'].astype(int) - cpu.seg_prob.astype(int))
  assert qd.max() <= 1 and (qd > 0).mean() < 1e-3, what                # expf vs scipy expit at bin edges
  assert dev['origins'] == [(k, tuple(v[0]), v[1]) for k, v in sorted(cpu.origins.items())], what
  assert dev['overlaps'] == sorted((k, int(i), int(c)) for k, v in cpu.overlaps.items()
                                   for i, c in zip(v[0], v[1])), what
  ctr = dev['ctr']
  assert ctr.inference_calls == cpu.counters['inference-calls'], what
  assert ctr.skip_threshold == cpu.counters['skip_threshold'], what
  assert ctr.skip_invalid_pos == cpu.counters['skip_invalid_pos'], what
  assert ctr.invalid_small == cpu.counters['invalid-small'], what
  assert ctr.invalid_weak == cpu.counters['invalid-weak'], what
  assert ctr.seed_got_too_weak == cpu.counters['seed_got_too_weak'], what
  assert ctr.segment_at_calls == cpu.counters['segment_at-calls'], what
  assert ctr.voxels_segmented == cpu.counters['voxels-segmented'], what
  assert ctr.voxels_overlapping == cpu.counters['voxels-overlapping'], what


@pytest.mark.parametrize('name', ['x9', 'x5'])
def test_flood_fill_equals_the_pure_oracle_and_the_reference(golden_dir, name):
  from ffn_b200 import _lib, engine as eng
  g = np.load(os.path.join(golden_dir, 'exact_flood_fill.npz'), allow_pickle=False)
  fov, deltas, depth, vol, seeds, opts = flood_case(g, name)
  w, b = xn.flood_net(depth)
  cpu = ff.Canvas(lambda s, im: xn.logits(w, b, s, im, 'fp32'), xn.flood_image_f32(vol), fov, deltas,
                  ff.Options(**opts))
  cpu.segment_all(seeds)
  np.testing.assert_array_equal(cpu.segmentation, g[name + '_segmentation'])   # the pure oracle is the reference
  want_ctr = json.loads(str(g[name + '_counters']))
  for mname, (mode, _) in _modes().items():
    e = eng.Engine(w, b, fov, deltas, compute_mode=mode)
    for chains in (1, 4):
      e.set_chains(chains)
      dev = _flood(e, vol, seeds, opts)
      what = '%s %s %d chains' % (name, mname, chains)
      _check_flood(dev, cpu, what)
      np.testing.assert_array_equal(dev['seed'], g[name + '_seed_canvas'], err_msg=what)
      assert dev['ctr'].inference_calls == want_ctr['inference-calls'], what
    # one object with segment_at, from the origin of the longest run
    e.set_chains(0)
    o = g[name + '_origins']
    start = tuple(int(v) for v in o[int(np.argmax(o[:, 4])), 1:4])
    cv = eng.DeviceCanvas(e, vol, eng.make_options(**{k: v for k, v in xn.FLOOD_OPTIONS.items()}),
                          xn.FLOOD_MEAN, xn.FLOOD_STDDEV)
    st = cv.segment_at(start)
    one = ff.Canvas(lambda s, im: xn.logits(w, b, s, im, 'fp32'), xn.flood_image_f32(vol), fov, deltas,
                    ff.Options(**xn.FLOOD_OPTIONS))
    assert st.iters == one.segment_at(start) and st.iters > 1, mname
    np.testing.assert_array_equal(cv.read(_lib.ARRAY_SEED), one.seed, err_msg=mname)
    cv.close()
    e.close()


def test_profiled_build_equals_the_plain_build(golden_dir):
  """enable_profiling switches every launch to the profiled instantiation (flood_profiled.cu): the same logits and
  the same flood fill bit for bit.  Its counters are non-negative, the conv layers take no longer than the kernel,
  and both consumer warpgroups report MMA and epilogue cycles in the fp16 mode."""
  from ffn_b200 import engine as eng
  g = np.load(os.path.join(golden_dir, 'exact_flood_fill.npz'), allow_pickle=False)
  fov_f, deltas_f, depth_f, vol, seeds_f, opts = flood_case(g, 'x9')
  wf, bf = xn.flood_net(depth_f)
  for case in ('fov9x17x25_d3', 'fov25x33x33_d4', 'fov9x17x25_depth16'):
    fov, depth, w, b, seeds, imgs = sweep_case(case)
    for mname, (mode, omode) in _modes().items():
      e = eng.Engine(w, b, fov, _deltas(fov), compute_mode=mode)
      e.enable_profiling(True)
      e.profile(reset=True)
      for chains in (1, 4):
        e.set_chains(chains)
        _assert_equal(e.predict(seeds, imgs), _want(w, b, seeds, imgs, omode),
                      'profiled %s %s chains %d' % (case, mname, chains))
      prof = e.profile(reset=True)
      for cta, c in prof.items():
        assert all(v >= 0 for v in c.values()), (case, mname, cta, c)
        assert c['conv_layers'] <= c['kernel'], (case, mname, cta, c)
        if mname == 'tc':
          for k in ('mma', 'mma_wg1', 'epi_body', 'epi_body_wg1'):
            assert c[k] > 0, (case, cta, k, c)
      e.close()
  for mname, (mode, _) in _modes().items():
    e = eng.Engine(wf, bf, fov_f, deltas_f, compute_mode=mode)
    plain = _flood(e, vol, seeds_f, opts)
    e.enable_profiling(True)
    prof = _flood(e, vol, seeds_f, opts)
    for k in ('seg', 'seed', 'qprob'):
      np.testing.assert_array_equal(prof[k], plain[k], err_msg='%s %s' % (mname, k))
    assert prof['origins'] == plain['origins'] and prof['overlaps'] == plain['overlaps'], mname
    c = e.profile(reset=True)['cta0']
    assert all(v >= 0 for v in c.values()) and c['steps'] > 0, (mname, c)
    e.close()


def test_flagship_geometry_hybrid_loop_checked_exactly():
  """fov (33, 33, 33), depth 12, deltas (8, 8, 8): the pure CPU loop is too slow here (seconds per float64 patch), so
  the device loop is compared with the hybrid oracle (the CPU loop driven by the device's predict), and every k-th
  patch the loop fed the network is checked against the float64 oracle, with the premise."""
  from ffn_b200 import _lib, engine as eng
  from ffn_b200.synthetic import voronoi_phantom
  fov, deltas, shape = (33, 33, 33), (8, 8, 8), (64, 72, 80)
  w, b = xn.flood_net(12)
  _, cells = voronoi_phantom(shape, seed=31, cell_volume=30000.0, return_cells=True)
  vol = xn.flood_image(cells, 31)
  seeds = ff.grid_seeds(shape, step=16, offsets=(0, 8))
  opts = dict(xn.FLOOD_OPTIONS, min_segment_size=500, min_boundary_dist=(1, 1, 1))
  for mname in ('tc', 'x2'):
    mode, omode = _modes()[mname]
    e = eng.Engine(w, b, fov, deltas, compute_mode=mode)
    dev = _flood(e, vol, seeds, opts)
    fed = []

    def net(s, im):
      fed.append((np.array(s), np.array(im)))
      return e.predict(s, im)

    hyb = ff.Canvas(net, xn.flood_image_f32(vol), fov, deltas, ff.Options(**opts))
    hyb.segment_all(seeds)
    _check_flood(dev, hyb, mname)
    assert len(fed) > 20 and max(o[2] for o in dev['origins']) > 5, (len(fed), dev['origins'])
    picks = fed[::max(1, len(fed) // 3)][:3]
    s = np.stack([p[0] for p in picks])
    im = np.stack([p[1] for p in picks])
    xn.assert_exact(w, b, s, im, omode)
    _assert_equal(e.predict(s, im), _want(w, b, s, im, omode), 'flagship %s' % mname)
    print('%s: %d steps, %d objects; %d patches checked exactly' % (mname, len(fed), len(dev['origins']), len(picks)))
    e.close()
