"""The example-loop oracle against the reference's own examples.py (tests/golden/examples_ref.npz), the thresholds'
float64 semantics, the seeded example stream and the TFRecord coordinate reader.  CPU only."""

import gzip
import os
import struct

import numpy as np
import pytest
from scipy import special

import examples_oracle as eo
from ffn_b200 import _lib
from ffn_b200.training import examples as ex
from ffn_b200.training import inputs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'examples_ref.npz')


def make_oracle(c):
  return eo.ExampleLoopOracle(c['volumes'], c['offset_scale'], c['fov'], c['deltas'], c['batch'], c['policy'],
                              c['fov_moves'], ex.seed_logits(0.05), ex.thresholds(c['threshold']), c['shifts'])


@pytest.mark.parametrize('i', range(len(eo.cases())))
def test_oracle_equals_reference(i):
  ref = np.load(GOLDEN)
  c = eo.case_setup(eo.cases()[i])
  o = make_oracle(c)
  coords = eo.as_coords(c['rows'])
  rng = np.random.RandomState(c['logit_seed'])
  pos = 0
  for step in range(eo.N_STEPS):
    seed, image, labels, offsets, example, taken = o.next(coords[pos:])
    pos += taken
    np.testing.assert_array_equal(offsets, ref['offsets_%d' % i][step], err_msg='step %d' % step)
    np.testing.assert_array_equal(example, ref['example_%d' % i][step], err_msg='step %d' % step)
    assert taken == ref['consumed_%d' % i][step]
    if step in eo.FULL_STEPS:
      for k, v in (('seed', seed), ('image', image), ('labels', labels)):
        np.testing.assert_array_equal(v, ref['%s_%d_%d' % (k, i, step)], err_msg='%s at step %d' % (k, step))
    o.update(eo.step_logits(rng, c))


@pytest.mark.parametrize('bug', ['valid', 'wanted', 'score'])
def test_float32_thresholds_change_the_fixture(bug):
  """Comparing a seed value, a label or a face maximum against the float32-rounded threshold instead of in float64
  changes the offsets of at least one fixture case, so neither the oracle nor the device can do it unseen."""
  ref = np.load(GOLDEN)
  changed = []
  for i, case in enumerate(eo.cases()):
    c = eo.case_setup(case)
    o = eo.ExampleLoopOracle(c['volumes'], c['offset_scale'], c['fov'], c['deltas'], c['batch'], c['policy'],
                             c['fov_moves'], ex.seed_logits(0.05), ex.thresholds(c['threshold']), c['shifts'],
                             f32=(bug,))
    coords = eo.as_coords(c['rows'])
    rng = np.random.RandomState(c['logit_seed'])
    pos, offsets = 0, []
    for _ in range(eo.N_STEPS):
      out = o.next(coords[pos:])
      pos += out[5]
      offsets.append(out[3])
      o.update(eo.step_logits(rng, c))
    if not np.array_equal(np.array(offsets), ref['offsets_%d' % i]):
      changed.append(case[0])
  assert changed, bug
  assert all(eo.case_setup(k)['snap'] for k in eo.cases() if k[0] in changed)


def test_snapped_thresholds_split_the_precisions():
  for t in (0.9499999, 0.7):
    s = ex.thresholds(t)[0]
    assert float(np.float32(s)) < s
  s, l = ex.thresholds(0.0500000023)
  assert float(np.float32(0.05)) < l and np.float32(l) == np.float32(0.05) and float(np.float32(s)) < s
  assert float(ex.seed_logits(0.05)[1]) >= s


def test_cases_cover_both_outcomes():
  ref = np.load(GOLDEN)
  for i, case in enumerate(eo.cases()):
    consumed = ref['consumed_%d' % i]
    offsets = ref['offsets_%d' % i].reshape(-1, 3)
    assert consumed[1:].sum() > 0, case[0]              # examples are exhausted and replaced
    assert (np.abs(offsets).sum(1) > 0).any(), case[0]  # and moves are taken
  assert any(np.min(np.stack([v[1] for v in eo.case_setup(c)['volumes']])) < 0 for c in eo.cases())


def test_thresholds_compare_in_float64():
  pad, centre = ex.seed_logits(0.05)
  assert centre == np.float32(special.logit(np.float32(0.95)))
  seed_thr, label_thr = ex.thresholds(0.95)
  assert float(centre) < seed_thr                       # a fresh seed fails 0.95: the reference would loop forever
  assert float(np.float32(0.95)) < label_thr            # and so does the 0.95f label
  seed_thr, label_thr = ex.thresholds(0.9499999)
  assert float(centre) >= seed_thr and float(np.float32(0.95)) >= label_thr
  assert float(pad) < ex.thresholds(0.05)[0] + 1e-6


def test_model_shifts_keep_duplicates():
  s = ex.model_shifts((0, 2, 3))
  assert len(s) == 24 and len(set(s)) == 8   # every (x, y, 0) three times, the origin never
  assert s[0] == (0, -2, -3) and ex.model_shifts((1, 1, 1))[0] == (-1, -1, -1)


def test_stream_is_seeded_and_draws_allowed_transforms():
  vols = np.array([0, 1, 1, 0, 2])
  centers = np.arange(15).reshape(5, 3)
  a = ex.ExampleStream(vols, centers, (1, 2), (0, 2), seed=3).take(23)
  b = ex.ExampleStream(vols, centers, (1, 2), (0, 2), seed=3).take(23)
  np.testing.assert_array_equal(a, b)
  assert a.dtype == _lib.EXAMPLE_COORD_DTYPE
  for epoch in range(4):
    assert sorted(a['center_xyz'][epoch * 5:epoch * 5 + 5, 0].tolist()) == [0, 3, 6, 9, 12]
  assert (a['permutation_zyx'][:, 0] == 0).all() and (a['reflect_zyx'][:, 1] == 0).all()
  assert {tuple(p) for p in a['permutation_zyx']} == {(0, 1, 2), (0, 2, 1)}
  assert a['reflect_zyx'][:, [0, 2]].any(0).all()


def _varint(v):
  v &= (1 << 64) - 1
  out = b''
  while True:
    b = v & 0x7F
    v >>= 7
    if v:
      out += bytes([b | 0x80])
    else:
      return out + bytes([b])


def _ld(field, payload):
  return _varint(field << 3 | 2) + _varint(len(payload)) + payload


def _example(center, name, packed=True):
  if packed:
    ints = _ld(1, b''.join(_varint(v) for v in center))
  else:
    ints = b''.join(_varint(1 << 3) + _varint(v) for v in center)
  feats = (_ld(1, _ld(1, b'center') + _ld(2, _ld(3, ints))) +
           _ld(1, _ld(1, b'label_volume_name') + _ld(2, _ld(1, _ld(1, name)))))
  return _ld(1, feats)


def test_tfrecord_reader(tmp_path):
  recs = [((5, 6, 7), b'vol', True), ((0, 2**40, -3), 'Zellkörper'.encode('utf-8'), False), ((1, 1, 1), b'b', True)]
  for k, chunk in enumerate((recs[:2], recs[2:])):
    with gzip.open(str(tmp_path / ('c%d.tfr' % k)), 'wb') as f:
      for center, name, packed in chunk:
        data = _example(center, name, packed)
        f.write(struct.pack('<Q', len(data)) + b'\0' * 4 + data + b'\0' * 4)
  centers, names = inputs.load_coordinates(str(tmp_path / 'c*.tfr'))
  np.testing.assert_array_equal(centers, [r[0] for r in recs])
  assert names == ['vol', 'Zellkörper', 'b']
  with pytest.raises(FileNotFoundError):
    inputs.load_coordinates(str(tmp_path / 'none*'))
