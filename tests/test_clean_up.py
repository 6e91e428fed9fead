"""Connected-component clean-up on the host: the oracle against the fixture written by the reference's own
clean_up / clean_up_and_count (tests/golden/make_golden_clean_up.py), the split_cc=False path, and the argument checks
that run before any device work."""
import ast
import os

import numpy as np
import pytest

from ffn_b200.inference import segmentation
from oracle import clean_up as ocu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'clean_up_ref.npz')
ERRORS = {'ValueError': ValueError, 'TypeError': TypeError}


def clean_up_cases():
  """One dict per fixture case: tag, fn, kwargs, seg, after, error, and per returned dict ('map', 'counts') its
  kind ('None' or 'dict'), sorted keys, values and their type names."""
  g = np.load(GOLDEN)
  out = []
  for i in range(int(g['n'])):
    c = {k: g['%s_%d' % (k, i)] for k in ('seg', 'after', 'map_keys', 'map_vals', 'counts_keys', 'counts_vals')}
    for k in ('tag', 'fn', 'error', 'map_kind', 'map_ktype', 'map_vtype', 'counts_kind', 'counts_ktype',
              'counts_vtype'):
      c[k] = str(g['%s_%d' % (k, i)])
    c['kwargs'] = dict(ast.literal_eval(str(g['kwargs_%d' % i])))
    out.append(c)
  return out


def call(module, case, seg):
  """Runs module.<fn>(seg, **kwargs); returns (id map, counts) as clean_up_and_count does."""
  res = getattr(module, case['fn'])(seg, **case['kwargs'])
  if case['fn'] == 'clean_up':
    return res, None
  return res


def check_result(case, seg, maps):
  tag = case['tag']
  assert seg.dtype == np.uint64 and np.array_equal(seg, case['after']), tag
  for name, d in zip(('map', 'counts'), maps):
    if case[name + '_kind'] == 'None':
      assert d is None, (tag, name)
      continue
    assert isinstance(d, dict), (tag, name)
    keys = sorted(d)
    assert np.array_equal(np.array(keys, np.uint64), case[name + '_keys']), (tag, name)
    vals = [d[k] for k in keys]
    assert np.array_equal(np.array(vals, case[name + '_vals'].dtype), case[name + '_vals']), (tag, name)
    assert {type(k).__name__ for k in keys} <= {case[name + '_ktype']}, (tag, name)
    assert {type(v).__name__ for v in vals} <= {case[name + '_vtype']}, (tag, name)


CASES = clean_up_cases()


def test_fixture_covers_the_cases():
  by_tag = {c['tag']: c for c in CASES}
  assert {c['error'] for c in CASES} == {'', 'ValueError'}
  # connectivity tells the diagonal, checkerboard and corner cases apart
  for stem in ('diagonal', 'checker3d', 'corner26'):
    sizes = [np.unique(by_tag['%s_c%d' % (stem, c)]['after']).size for c in (1, 2, 3)]
    assert sizes[0] > sizes[1] or sizes[1] > sizes[2], stem
  # a dusted voxel comes before the first input zero, so 0 maps to the dusted id
  c = by_tag['dust_before_zero']
  assert c['seg'].ravel()[0] == 8 and c['after'].ravel()[0] == 0 and c['map_keys'][0] == 0 and c['map_vals'][0] == 8
  assert c['map_ktype'] == c['map_vtype'] == 'uint64' and c['counts_vtype'] == 'int64'
  assert by_tag['ids_ge_2_63']['seg'].max() >= 2**63 and by_tag['ids_ge_2_32']['seg'].max() >= 2**32
  assert by_tag['empty']['map_kind'] == 'dict' and by_tag['empty']['map_keys'].size == 0
  assert not by_tag['one_id_min_drop']['after'].any()


@pytest.mark.parametrize('case', CASES, ids=lambda c: c['tag'])
def test_oracle_equals_reference(case):
  seg = case['seg'].copy()
  if case['error']:
    with pytest.raises(ERRORS[case['error']]):
      call(ocu, case, seg)
    return
  check_result(case, seg, call(ocu, case, seg))


@pytest.mark.parametrize('case', [c for c in CASES if c['kwargs'].get('split_cc') is False or not c['seg'].any()],
                         ids=lambda c: c['tag'])
def test_host_paths_equal_reference(case):
  """split_cc=False, all-zero and empty input never reach the device."""
  seg = case['seg'].copy()
  check_result(case, seg, call(segmentation, case, seg))


@pytest.mark.parametrize('case', [c for c in CASES if c['error']], ids=lambda c: c['tag'])
def test_connectivity_errors_decided_on_the_host(case):
  with pytest.raises(ERRORS[case['error']]):
    call(segmentation, case, case['seg'].copy())


@pytest.mark.parametrize('dtype', [np.uint32, np.int64, np.uint8])
def test_dtype_error_decided_on_the_host(dtype):
  seg = np.ones((2, 3, 4), dtype)
  for fn in (segmentation.clean_up, segmentation.clean_up_and_count):
    with pytest.raises(TypeError):
      fn(seg)
  with pytest.raises(ValueError):
    segmentation.clean_up(np.ones((2, 2, 2, 2), np.uint64))


def test_ffn_namespace_alias():
  from ffn.inference import segmentation as alias
  assert alias is segmentation
  assert callable(alias.clean_up) and callable(alias.clean_up_and_count)
