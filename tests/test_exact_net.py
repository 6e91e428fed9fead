"""Exactly representable networks (oracle/exact_net.py) on the CPU: the premise, the oracles and the power of an
exact comparison.

* Every network and input tests/test_gpu_exact_net.py runs satisfies the premise in the modes it is run in, so the
  device must equal the float64 oracle (fp16 mode: the float64 fp16-operand oracle) with assert_array_equal.
* Under the premise the float64 oracle and torch's float32 CPU conv stack give identical logits.
* Each deliberate bug changes at least one logit of its probe, so an exact comparison catches it: among them the
  three that pass the tolerance tests (the residual stream or the biases rounded to fp16, the seed operand left
  unrounded), the wrong rounding mode, a flushed subnormal, an unmasked dx tap, a dy tap read across z-planes, a bias
  on the wrong channel and b_lom added twice.
* The flood-fill oracle loop driven by the float64 flood network reproduces the reference's own segment_all
  (tests/golden/make_golden_exact.py) bit for bit, and that run reaches the tie rules: faces with equal maxima and
  logits exactly on the thresholds.

EXACT_SWEEP and the inputs are defined here and shared with the GPU test.
"""

import json
import os

import numpy as np
import pytest

from oracle import exact_net as xn
from oracle import flood_fill as ff
from test_geometry_oracle import SWEEP, _check_canvas, rowspace_logits

# (id, fov, depth, batch): every SWEEP geometry at its depth, and depths 1, 2, 12 and 16 at fov (9, 17, 25).  Small
# fields of view run batches of 1, 4, 5 and 9 patches (9 crosses two four-patch chain multiplexes).
EXACT_SWEEP = [(case, fov, depth, 1 if np.prod(fov) > 20000 else 5) for case, fov, depth, _ in SWEEP] + [
    ('fov9x17x25_depth%d' % d, (9, 17, 25), d, n) for d, n in ((1, 9), (2, 4), (12, 1), (16, 4))]


def sweep_case(case):
  _, fov, depth, n = next(c for c in EXACT_SWEEP if c[0] == case)
  w, b = xn.random_net(depth, 100 + depth)
  seeds, imgs = xn.random_patches(fov, n, int(np.prod(fov)) % 9973 + depth)
  return fov, depth, w, b, seeds, imgs


PROBE_FOV = (9, 17, 25)


# ------------------------------------------------------------------------------------------------------------------
# The premise and the two oracles
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('case', [c[0] for c in EXACT_SWEEP])
def test_premise_holds_for_the_gpu_sweep(case):
  fov, depth, w, b, seeds, imgs = sweep_case(case)
  for mode in ('fp16', 'x2', 'fp32'):
    assert xn.premise_margin(w, b, seeds, imgs, mode) > 1.0, (case, mode)
  good = xn.logits(w, b, seeds, imgs, 'fp32')
  assert (good != seeds).mean() > 0.9          # the network moves nearly every logit


@pytest.mark.parametrize('name', sorted(xn.PROBES))
def test_premise_holds_for_every_probe(name):
  w, b, seeds, imgs = xn.PROBES[name](PROBE_FOV)
  for mode in ('fp16', 'x2', 'fp32'):
    assert xn.premise_margin(w, b, seeds, imgs, mode) > 1.0, (name, mode)


def test_premise_checker_rejects_what_it_must():
  w, b = xn.random_net(2, 102)
  seeds, imgs = xn.random_patches((5, 7, 9), 1, 3)
  xn.assert_exact(w, b, seeds, imgs, 'x2')
  bad = np.array(imgs)
  bad.reshape(-1)[0] = 1.0 + 2.0 ** -20            # operand with a lo part that is not an fp16 number
  with pytest.raises(xn.PremiseError):
    xn.assert_exact(w, b, seeds, bad, 'x2')
  w2 = [np.array(x) for x in w]
  w2[2].reshape(-1)[np.flatnonzero(w2[2])[0]] = 1.0 + 2.0 ** -11   # weight not fp16-exact
  with pytest.raises(xn.PremiseError):
    xn.assert_exact(w2, b, seeds, imgs, 'fp32')
  big = np.array(imgs) * np.float32(2.0 ** 12)     # sums past 2^(24-q)
  big.reshape(-1)[0] = 2.0 ** -8
  with pytest.raises(xn.PremiseError):
    xn.assert_exact(w, b, seeds, big, 'fp32')


@pytest.mark.parametrize('case', ['fov9x17x25_d3', 'fov11x13x15_d6_random', 'fov9x17x25_d16'])
def test_float32_oracle_equals_float64(case):
  fov, depth, w, b, seeds, imgs = sweep_case(case)
  for mode in ('fp32', 'fp16'):
    np.testing.assert_array_equal(xn.logits_f32(w, b, seeds, imgs, mode), xn.logits(w, b, seeds, imgs, mode))
  for name, make in xn.PROBES.items():
    pw, pb, ps, pi = make(PROBE_FOV)
    for mode in ('fp32', 'fp16'):
      np.testing.assert_array_equal(xn.logits_f32(pw, pb, ps, pi, mode), xn.logits(pw, pb, ps, pi, mode),
                                    err_msg='%s %s' % (name, mode))


def test_fp16_rounding_helpers():
  x = np.asarray([2049.0, 2051.0, -2049.0, 2050.0, 1000.25, 2.0 ** -25, 3 * 2.0 ** -25, 2.0 ** -15])
  np.testing.assert_array_equal(xn.round_f16(x), [2048, 2052, -2048, 2050, 1000.0, 0.0, 2.0 ** -23, 2.0 ** -15])
  np.testing.assert_array_equal(xn.round_f16(x, 'rtz'), [2048, 2050, -2048, 2050, 1000.0, 0.0, 2.0 ** -24, 2.0 ** -15])
  np.testing.assert_array_equal(xn.round_f16(x, 'rha'), [2050, 2052, -2050, 2050, 1000.5, 2.0 ** -24, 2.0 ** -23,
                                                         2.0 ** -15])
  np.testing.assert_array_equal(xn.round_f16(x, flush=True)[-1], 0.0)
  assert xn.frac_bits([0.75, 3.0, -0.125]) == 3 and xn.frac_bits([0.0, 4.0]) == 0 and xn.frac_bits([2.0 ** -24]) == 24


# ------------------------------------------------------------------------------------------------------------------
# Every bug changes a logit
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('name', sorted(xn.PROBES))
def test_probe_catches_its_bugs(name):
  w, b, seeds, imgs = xn.PROBES[name](PROBE_FOV)
  for bug, mode in xn.PROBE_BUGS[name]:
    good = xn.logits(w, b, seeds, imgs, mode)
    bad = xn.logits(w, b, seeds, imgs, mode, bug)
    assert not np.array_equal(good, bad), (name, bug, mode)
    print(name, bug, mode, '%d logits differ, max %.3g' % ((good != bad).sum(), np.abs(good - bad).max()))


def test_rounding_modes_give_three_different_answers():
  w, b, seeds, imgs = xn.probe_rounding(PROBE_FOV)
  rne, rtz, rha = (xn.logits(w, b, seeds, imgs, 'fp16', bug) for bug in (None, 'round_toward_zero',
                                                                           'round_half_away'))
  assert not np.array_equal(rne, rtz) and not np.array_equal(rne, rha) and not np.array_equal(rtz, rha)
  # the fp32 and split modes carry the odd integers unrounded
  np.testing.assert_array_equal(xn.logits(w, b, seeds, imgs, 'fp32'), 2 * imgs + 1 - 2048 + seeds)


@pytest.mark.parametrize('case', ['fov3_d1', 'fov9x17x3_d2', 'fov9x17x25_d3', 'fov11x13x15_d6_random'])
def test_structural_bugs_change_a_logit_of_the_random_nets(case):
  """The row-space restatement of test_geometry_oracle.py (float64, no operand rounding) on the random exact
  networks: without a bug it is the oracle bit for bit; each bug changes at least one logit."""
  fov, depth, w, b, seeds, imgs = sweep_case(case)
  good = xn.logits(w, b, seeds[0], imgs[0], 'fp32')
  np.testing.assert_array_equal(rowspace_logits(w, b, seeds[0], imgs[0]).astype(np.float32), good)
  for kw in (dict(x_mask=False), dict(zero_line=False), dict(lom_bias_twice=True)):
    bad = rowspace_logits(w, b, seeds[0], imgs[0], **kw).astype(np.float32)
    assert not np.array_equal(bad, good), (case, kw)
  for bug in ('bias_wrong_channel', 'lom_bias_twice'):   # (their values are fp16-exact: the probes cover the rest)
    assert not np.array_equal(xn.logits(w, b, seeds[0], imgs[0], 'fp32', bug), good), (case, bug)


# ------------------------------------------------------------------------------------------------------------------
# The flood fill under the flood network
# ------------------------------------------------------------------------------------------------------------------

def flood_case(g, name):
  p = name + '_'
  fov, deltas = tuple(int(v) for v in g[p + 'fov']), tuple(int(v) for v in g[p + 'deltas'])
  opts = dict(xn.FLOOD_OPTIONS, min_segment_size=int(g[p + 'min_segment_size']),
              min_boundary_dist=tuple(int(v) for v in g[p + 'min_boundary_dist']))
  return fov, deltas, int(g[p + 'depth']), g[p + 'volume'], g[p + 'seeds'], opts


@pytest.mark.parametrize('name', ['x9', 'x5'])
def test_exact_flood_fill_bit_exact_vs_reference(golden_dir, name):
  g = np.load(os.path.join(golden_dir, 'exact_flood_fill.npz'), allow_pickle=False)
  fov, deltas, depth, vol, seeds, opts = flood_case(g, name)
  w, b = xn.flood_net(depth)
  assert vol.dtype == np.uint8
  canvas = ff.Canvas(lambda s, im: xn.logits(w, b, s, im, 'fp32'), xn.flood_image_f32(vol), fov, deltas,
                     ff.Options(**opts))
  canvas.segment_all(seeds)
  _check_canvas(canvas, g, name + '_')
  assert canvas.min_margin == 0.0                                      # a decision sat exactly on a threshold
  ties = json.loads(str(g[name + '_ties']))
  assert ties['face_ties'] > 0 and ties['threshold_hits'] > 0, ties
  assert max(int(v) for v in g[name + '_origins'][:, 4]) > 10           # an object grows


@pytest.mark.parametrize('name', ['x9', 'x5'])
def test_flood_network_premise_along_the_fixture_run(golden_dir, name):
  """Every patch the run feeds the network satisfies the premise in all three modes, and the fp16-operand oracle
  equals the float64 one there (every seed the loop feeds back is fp16-exact): one expected answer for every mode."""
  g = np.load(os.path.join(golden_dir, 'exact_flood_fill.npz'), allow_pickle=False)
  fov, deltas, depth, vol, seeds, opts = flood_case(g, name)
  w, b = xn.flood_net(depth)
  patches = []

  def net(s, im):
    patches.append((np.array(s), np.array(im)))
    return xn.logits(w, b, s, im, 'fp32')

  canvas = ff.Canvas(net, xn.flood_image_f32(vol), fov, deltas, ff.Options(**opts))
  canvas.segment_all(seeds)
  s = np.stack([p[0] for p in patches])
  im = np.stack([p[1] for p in patches])
  for mode in ('fp16', 'x2', 'fp32'):
    assert xn.premise_margin(w, b, s, im, mode) > 1.0, mode
  np.testing.assert_array_equal(xn.logits(w, b, s, im, 'fp16'), xn.logits(w, b, s, im, 'fp32'))
