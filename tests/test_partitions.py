"""Partition map (compute_partitions.py:115-204): the numpy oracle against the reference's own function
(tests/golden/partitions_ref.npz, from make_golden_partitions.py), and the host-side argument checks of
ffn_b200.partitions and of the compute_partitions.py script, none of which needs a device."""

import os

import numpy as np
import pytest
from google.protobuf import text_format

import compute_partitions as script
from ffn_b200 import _lib
from ffn_b200 import partitions
from ffn_b200.inference import inference_pb2
from ffn_b200.inference import storage
from oracle import partitions as op

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'partitions_ref.npz')
ERRORS = {'IndexError': IndexError, 'ValueError': ValueError, 'TypeError': TypeError, 'OverflowError': OverflowError}


def fixture():
  return np.load(GOLDEN)


def reference_cases(tmp_dir):
  """One dict per fixture case: the reference's arguments (mask_configs parsed, a volume mask written to tmp_dir)
  and what it returned or raised."""
  g = fixture()
  out = []
  for i in range(int(g['n_cases'])):
    regions = None
    if g['has_regions_%d' % i]:
      regions = [tuple(int(v) if is_int else float(v) for v, is_int in zip(row, ints))
                 for row, ints in zip(g['regions_%d' % i], g['regions_int_%d' % i])]
    text = str(g['mask_text_%d' % i])
    mask_configs = None
    if text:
      if g['has_mask_volume_%d' % i]:
        path = os.path.join(str(tmp_dir), 'mask_%d.npy' % i)
        np.save(path, g['mask_volume_%d' % i])
        text = text.replace(str(g['mask_placeholder']), path + ':')
      mask_configs = inference_pb2.MaskConfigs()
      text_format.Parse(text, mask_configs)
    out.append({
        'tag': str(g['tag_%d' % i]), 'seg': g['seg_%d' % i], 'thresholds': g['thresholds_%d' % i].tolist(),
        'lom_radius': [int(v) for v in g['lom_radius_%d' % i]],
        'id_whitelist': [int(w) for w in g['whitelist_%d' % i]] if g['has_whitelist_%d' % i] else None,
        'exclusion_regions': regions, 'mask_configs': mask_configs, 'min_size': int(g['min_size_%d' % i]),
        'error': str(g['error_%d' % i]), 'corner': g['corner_%d' % i], 'out': g['out_%d' % i],
        'seg_after': g['seg_after_%d' % i]})
  return out


def case_ids():
  g = fixture()
  return [str(g['tag_%d' % i]) for i in range(int(g['n_cases']))]


def call(fn, c, **kw):
  """fn(...) on a copy of the case's volume -> (volume after the call, result or the exception's name)."""
  seg = c['seg'].copy()
  try:
    return seg, fn(seg, c['thresholds'], c['lom_radius'], c['id_whitelist'], c['exclusion_regions'],
                   c['mask_configs'], c['min_size'], **kw)
  except (IndexError, ValueError, TypeError, OverflowError) as e:
    return seg, type(e).__name__


def oracle_fn(seg, thresholds, lom_radius, id_whitelist, exclusion_regions, mask_configs, min_size):
  mask = None
  if mask_configs is not None:
    mask = storage.build_mask(mask_configs.masks, (0, 0, 0), seg.shape)
  return op.compute_partitions(seg, thresholds, lom_radius, id_whitelist, exclusion_regions, mask, min_size)


def assert_matches(c, seg, res):
  assert seg.dtype == c['seg_after'].dtype and (seg == c['seg_after']).all(), c['tag']
  if c['error']:
    assert res == c['error'], (c['tag'], res)
    return
  corner, out = res
  assert (np.asarray(corner) == c['corner']).all(), c['tag']
  assert out.dtype == np.uint8 and out.shape == c['out'].shape, (c['tag'], out.shape)
  assert (out == c['out']).all(), (c['tag'], int((out != c['out']).sum()))


def test_fixture_covers_the_cases():
  tags = case_ids()
  for t in ('iso', 'aniso', 'zero_x', 'unsorted', 'single', 'min1', 'min_drop', 'whitelist', 'excl_int', 'excl_float',
            'mask_expr', 'mask_volume', 'u64_big', 'i64_neg', 'all_zero', 'one_label', 'smaller_than_lom',
            'empty_thresholds'):
    assert t in tags
  g = fixture()
  assert g['main_out'].dtype == np.uint8 and g['main_partition_counts'].shape[0] == 2


@pytest.mark.parametrize('idx', range(len(case_ids())), ids=case_ids())
def test_oracle_equals_reference(idx, tmp_path):
  c = reference_cases(tmp_path)[idx]
  seg, res = call(oracle_fn, c)
  assert_matches(c, seg, res)


@pytest.fixture
def no_device(monkeypatch):
  def refuse():
    raise AssertionError('the library was loaded')
  monkeypatch.setattr(_lib, 'load', refuse)


SEG = np.arange(4 * 5 * 6, dtype=np.int32).reshape(4, 5, 6) % 7


@pytest.mark.parametrize('kwargs,exc', [
    (dict(seg_array=SEG.astype(np.float32)), TypeError),
    (dict(seg_array=SEG.astype(bool)), TypeError),
    (dict(seg_array=SEG[0]), ValueError),
    (dict(seg_array=SEG[None]), ValueError),
    (dict(lom_radius=[1, -1, 1]), ValueError),
    (dict(lom_radius=[1, 1]), ValueError),
    (dict(lom_radius=[1, 1.5, 1]), TypeError),
    (dict(thresholds=['a']), ValueError),
    (dict(exclusion_regions=[(1, 2, 3)]), ValueError),
    (dict(exclusion_regions=[(1, 2, 3, 'r')]), TypeError),
])
def test_host_argument_errors(no_device, kwargs, exc):
  args = dict(seg_array=SEG.copy(), thresholds=[0.5], lom_radius=[1, 1, 1], min_size=0)
  args.update(kwargs)
  with pytest.raises(exc):
    partitions.compute_partitions(**args)


def test_too_many_voxels(no_device):
  big = np.lib.stride_tricks.as_strided(np.zeros(1, np.uint8), shape=(1024, 1024, 2048), strides=(0, 0, 0))
  with pytest.raises(ValueError, match='2\\^31'):
    partitions.compute_partitions(big, [0.5], [1, 1, 1])


def test_whitelist_by_value():
  bits = partitions._whitelist_bits([3, 3.0, 2.5, '4', -1, 2**63, np.uint64(7), True], np.uint64)
  assert bits.tolist() == [1, 3, 7, 2**63]
  bits = partitions._whitelist_bits([-1, -2**63, 2**63, 300], np.int8)
  assert bits.tolist() == [2**64 - 1]


def test_partition_counts():
  hist = np.zeros(256, np.int64)
  hist[[0, 5, 255]] = [4, 2, 9]
  got = partitions.partition_counts(hist)
  want = np.array(np.unique(np.repeat(np.array([0, 5, 255], np.uint8), [4, 2, 9]), return_counts=True))
  assert got.shape == want.shape and (got == want).all()


def test_script_flag_parsing():
  assert script.parse_exclusion_regions(None) is None
  regions = script.parse_exclusion_regions(['1', '2', '3', '4', '1.5', '-2', '0', '2.25'])
  assert regions == [(1, 2, 3, 4), (1.5, -2, 0, 2.25)]
  assert [type(v) for v in regions[1]] == [float, int, int, float]
  with pytest.raises(ValueError):
    script.parse_exclusion_regions(['1', '2', '3'])
  configs = script.parse_mask_configs('masks { coordinate_expression { expression: "x > 3" } }')
  assert configs.masks[0].coordinate_expression.expression == 'x > 3'
  assert script.parse_mask_configs(None) is None


def test_script_layout_with_oracle(tmp_path, monkeypatch):
  """The script's input, bounding-box and output handling around the oracle reproduce the reference's `main`."""
  def oracle_map(seg, thresholds, lom_radius, id_whitelist, exclusion_regions, mask_configs, min_size, device):
    corner, out = oracle_fn(seg, thresholds, lom_radius, id_whitelist, exclusion_regions, mask_configs, min_size)
    return partitions.PartitionMap(corner, out, np.bincount(out.ravel(), minlength=256).astype(np.int64))
  monkeypatch.setattr(partitions, 'partition_map', oracle_map)
  g = fixture()
  src, dst = tmp_path / 'in.npz', tmp_path / 'out.npz'
  np.savez(src, **{'stack': g['main_seg'], 'stack.bounding_boxes': g['main_bboxes']})
  argv = [a.replace('in.h5:', '%s:' % src).replace('out.h5:', '%s:' % dst) for a in g['main_argv'].tolist()]
  script.FLAGS(['compute_partitions.py'] + argv)
  script.main([])
  with np.load(dst) as f:
    assert f['af'].dtype == np.uint8 and (f['af'] == g['main_out']).all()
    assert (f['af.bounding_boxes'] == g['main_out_bboxes']).all()
    assert (f['af.partition_counts'] == g['main_partition_counts']).all()
